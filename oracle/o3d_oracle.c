/*
 * o3d_oracle.c -- CPU ORACLE (test infrastructure, NOT product code).
 *
 * A plain-C, fp64 restatement of the reference hot path of
 * leggedrobotics/open3d_slam: the Open3D v0.15.1 routines it calls
 * (open3d_catkin/CMakeLists.txt:117-118 pins the tag) plus open3d_slam's own
 * croppers / transform / map-fusion / dense-map code.
 *
 * PARITY UNPINNED: the reference holds no test, golden vector or fixture on
 * this path (SURVEY.md section 4) and Open3D itself is neither under /root/reference
 * nor installable here, so the [O3D] parts below are restated from the
 * published v0.15.1 algorithm and cross-checked only against an independent
 * numpy/scipy restatement (oracle/np_oracle.py) and analytic known answers.
 *
 * Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline /
 * --impl reference legs may call into this file.  The product
 * (open3d_slam_b200/csrc) never links or loads it.
 *
 * Each function cites the reference file:line (relative to
 * /root/reference/open3d_slam/open3d_slam/, abbreviated core/) or the upstream
 * Open3D file it follows ([O3D] cpp/open3d/...).
 *
 * Deterministic choices made where the reference is unspecified:
 *   - hash-map iteration order  -> first-touch order of the voxel
 *   - exact distance ties       -> lowest point index wins (nanoflann: unspecified)
 *   - RandomDownSample seed     -> counter hash of (seed, index) (reference: random_device)
 *   - OpenMP reduction order    -> fixed 1024-element chunks summed in index order
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#include <stdio.h>
#ifdef _OPENMP
#include <omp.h>
#endif

#define ORC_EXPORT __attribute__((visibility("default")))

/* ------------------------------------------------------------------------- */
/*  small helpers                                                             */
/* ------------------------------------------------------------------------- */
static inline double sq(double x) { return x * x; }

/* nanoflann L2_Simple_Adaptor accumulates (dx*dx + dy*dy) + dz*dz */
static inline double dist2(const double* a, const double* b) {
  double dx = a[0] - b[0], dy = a[1] - b[1], dz = a[2] - b[2];
  return dx * dx + dy * dy + dz * dz;
}

/* ------------------------------------------------------------------------- */
/*  KD-tree (stands in for [O3D] KDTreeFlann / nanoflann, leaf size 15)       */
/*  exact k-NN; ties broken towards the lower index                           */
/* ------------------------------------------------------------------------- */
typedef struct {
  int left, right;   /* children (node ids) or -1 */
  int lo, hi;        /* point range [lo,hi) in perm for leaves */
  int dim;           /* split dimension */
  double split_lo;   /* max of left child along dim  */
  double split_hi;   /* min of right child along dim */
} kd_node;

typedef struct {
  const double* pts; /* n x 3 */
  int n;
  int* perm;
  kd_node* nodes;
  int n_nodes, cap_nodes;
  double bb_min[3], bb_max[3];
} kd_tree;

#define KD_LEAF 15

static int kd_new_node(kd_tree* t) {
  if (t->n_nodes == t->cap_nodes) {
    t->cap_nodes = t->cap_nodes ? 2 * t->cap_nodes : 1024;
    t->nodes = (kd_node*)realloc(t->nodes, sizeof(kd_node) * (size_t)t->cap_nodes);
  }
  return t->n_nodes++;
}

/* quickselect on perm[lo,hi) by coordinate dim so that perm[mid] is the median */
static void kd_select(kd_tree* t, int lo, int hi, int mid, int dim) {
  const double* P = t->pts;
  int* a = t->perm;
  while (hi - lo > 1) {
    /* median of three pivot */
    int m = lo + (hi - lo) / 2;
    double v0 = P[3 * a[lo] + dim], v1 = P[3 * a[m] + dim], v2 = P[3 * a[hi - 1] + dim];
    double pv = (v0 < v1) ? ((v1 < v2) ? v1 : (v0 < v2 ? v2 : v0)) : ((v0 < v2) ? v0 : (v1 < v2 ? v2 : v1));
    int i = lo, j = hi - 1;
    while (i <= j) {
      while (P[3 * a[i] + dim] < pv) i++;
      while (P[3 * a[j] + dim] > pv) j--;
      if (i <= j) {
        int tmp = a[i]; a[i] = a[j]; a[j] = tmp;
        i++; j--;
      }
    }
    if (mid <= j) hi = j + 1;
    else if (mid >= i) lo = i;
    else return;
  }
}

static int kd_build_rec(kd_tree* t, int lo, int hi) {
  int id = kd_new_node(t);
  kd_node nd;
  nd.left = nd.right = -1; nd.lo = lo; nd.hi = hi; nd.dim = 0; nd.split_lo = nd.split_hi = 0;
  if (hi - lo <= KD_LEAF) { t->nodes[id] = nd; return id; }
  double mn[3] = {INFINITY, INFINITY, INFINITY}, mx[3] = {-INFINITY, -INFINITY, -INFINITY};
  for (int i = lo; i < hi; i++) {
    const double* p = t->pts + 3 * t->perm[i];
    for (int d = 0; d < 3; d++) { if (p[d] < mn[d]) mn[d] = p[d]; if (p[d] > mx[d]) mx[d] = p[d]; }
  }
  int dim = 0; double ext = mx[0] - mn[0];
  for (int d = 1; d < 3; d++) if (mx[d] - mn[d] > ext) { ext = mx[d] - mn[d]; dim = d; }
  if (!(ext > 0.0)) { t->nodes[id] = nd; return id; } /* all identical: keep as (big) leaf */
  int mid = lo + (hi - lo) / 2;
  kd_select(t, lo, hi, mid, dim);
  double slo = -INFINITY, shi = INFINITY;
  for (int i = lo; i < mid; i++) { double v = t->pts[3 * t->perm[i] + dim]; if (v > slo) slo = v; }
  for (int i = mid; i < hi; i++) { double v = t->pts[3 * t->perm[i] + dim]; if (v < shi) shi = v; }
  nd.dim = dim; nd.split_lo = slo; nd.split_hi = shi;
  t->nodes[id] = nd;
  int l = kd_build_rec(t, lo, mid);
  int r = kd_build_rec(t, mid, hi);
  t->nodes[id].left = l; t->nodes[id].right = r;
  return id;
}

static kd_tree* kd_build(const double* pts, int n) {
  kd_tree* t = (kd_tree*)calloc(1, sizeof(kd_tree));
  t->pts = pts; t->n = n;
  t->perm = (int*)malloc(sizeof(int) * (size_t)(n > 0 ? n : 1));
  for (int i = 0; i < n; i++) t->perm[i] = i;
  for (int d = 0; d < 3; d++) { t->bb_min[d] = INFINITY; t->bb_max[d] = -INFINITY; }
  for (int i = 0; i < n; i++) for (int d = 0; d < 3; d++) {
    double v = pts[3 * i + d];
    if (v < t->bb_min[d]) t->bb_min[d] = v;
    if (v > t->bb_max[d]) t->bb_max[d] = v;
  }
  if (n > 0) kd_build_rec(t, 0, n);
  return t;
}

static void kd_free(kd_tree* t) {
  if (!t) return;
  free(t->perm); free(t->nodes); free(t);
}

/* result set: sorted ascending by (d2, idx), capacity k */
typedef struct { double* d2; int* idx; int k; int cnt; } kd_result;

static inline int kd_less(double da, int ia, double db, int ib) { return da < db || (da == db && ia < ib); }

static inline double kd_worst(const kd_result* r) { return r->cnt < r->k ? INFINITY : r->d2[r->k - 1]; }

static void kd_insert(kd_result* r, double d, int idx) {
  int i;
  if (r->cnt < r->k) i = r->cnt++;
  else {
    if (!kd_less(d, idx, r->d2[r->k - 1], r->idx[r->k - 1])) return;
    i = r->k - 1;
  }
  while (i > 0 && kd_less(d, idx, r->d2[i - 1], r->idx[i - 1])) {
    r->d2[i] = r->d2[i - 1]; r->idx[i] = r->idx[i - 1]; i--;
  }
  r->d2[i] = d; r->idx[i] = idx;
}

static void kd_search_rec(const kd_tree* t, int id, const double* q, kd_result* r, double* off, double mindist2) {
  const kd_node* nd = &t->nodes[id];
  if (nd->left < 0) {
    for (int i = nd->lo; i < nd->hi; i++) {
      int pi = t->perm[i];
      double d = dist2(q, t->pts + 3 * pi);
      kd_insert(r, d, pi);
    }
    return;
  }
  int dim = nd->dim;
  double v = q[dim];
  double dl = v - nd->split_lo; if (dl < 0) dl = 0; /* distance along dim to the left child's extent  */
  double dr = nd->split_hi - v; if (dr < 0) dr = 0; /* distance along dim to the right child's extent */
  int first, second; double cut;
  if (dl <= dr) { first = nd->left; second = nd->right; cut = dr; }
  else { first = nd->right; second = nd->left; cut = dl; }
  kd_search_rec(t, first, q, r, off, mindist2);
  double old = off[dim];
  if (cut < old) cut = old;
  double nmin = mindist2 - old * old + cut * cut;
  /* <= so that equal-distance points with a lower index are still seen */
  if (nmin <= kd_worst(r)) {
    off[dim] = cut;
    kd_search_rec(t, second, q, r, off, nmin);
    off[dim] = old;
  }
}

/* exact k nearest neighbours, sorted by (d2, idx). returns count */
static int kd_knn(const kd_tree* t, const double* q, int k, double* d2, int* idx) {
  kd_result r; r.d2 = d2; r.idx = idx; r.k = k; r.cnt = 0;
  if (t->n == 0 || k <= 0) return 0;
  double off[3]; double md = 0.0;
  for (int d = 0; d < 3; d++) {
    off[d] = 0.0;
    if (q[d] < t->bb_min[d]) off[d] = t->bb_min[d] - q[d];
    if (q[d] > t->bb_max[d]) off[d] = q[d] - t->bb_max[d];
    md += off[d] * off[d];
  }
  kd_search_rec(t, 0, q, &r, off, md);
  return r.cnt;
}

/* [O3D] KDTreeFlann::SearchHybrid (cpp/open3d/geometry/KDTreeFlann.cpp):
 * knnSearch(max_nn) then keep the prefix with d2 < radius*radius (lower_bound). */
static int kd_search_hybrid(const kd_tree* t, const double* q, double radius, int max_nn, double* d2, int* idx) {
  int k = kd_knn(t, q, max_nn, d2, idx);
  double r2 = radius * radius;
  int c = 0;
  while (c < k && d2[c] < r2) c++;
  return c;
}

/* exported thin wrappers so tests can exercise the tree directly */
ORC_EXPORT void* orc_kdtree_build(const double* pts, int n) { return kd_build(pts, n); }
ORC_EXPORT void orc_kdtree_free(void* t) { kd_free((kd_tree*)t); }
ORC_EXPORT int orc_kdtree_search_hybrid(void* t, const double* q, double radius, int max_nn, double* d2, int* idx) {
  return kd_search_hybrid((kd_tree*)t, q, radius, max_nn, d2, idx);
}

/* ------------------------------------------------------------------------- */
/*  P1  croppers        core/src/croppers.cpp:76-106 (crop), :121-165 (predicates) */
/* ------------------------------------------------------------------------- */
enum { ORC_CROP_NONE = 0, ORC_CROP_MAX_RADIUS = 1, ORC_CROP_MIN_RADIUS = 2, ORC_CROP_MINMAX_RADIUS = 3, ORC_CROP_CYLINDER = 4 };

typedef struct {
  int32_t kind;
  int32_t invert;            /* CroppingVolume::isInvertVolume_ (croppers.cpp:57-59) */
  double rmin, rmax, zmin, zmax;
  double center[3];          /* pose_.translation(); only the translation is used */
} orc_cropper;

static int orc_within_impl(const orc_cropper* c, const double* p) {
  double dx = p[0] - c->center[0], dy = p[1] - c->center[1], dz = p[2] - c->center[2];
  switch (c->kind) {
    case ORC_CROP_NONE: return 1;                                   /* croppers.cpp:53-55 */
    case ORC_CROP_MAX_RADIUS: return sqrt(dx * dx + dy * dy + dz * dz) <= c->rmax;    /* :136-138 */
    case ORC_CROP_MIN_RADIUS: return sqrt(dx * dx + dy * dy + dz * dz) >= c->rmin;    /* :149-151 */
    case ORC_CROP_MINMAX_RADIUS: { double d = sqrt(dx * dx + dy * dy + dz * dz); return d <= c->rmax && d >= c->rmin; } /* :121-124 */
    case ORC_CROP_CYLINDER: return p[2] >= c->zmin && p[2] <= c->zmax && sqrt(dx * dx + dy * dy) <= c->rmax; /* :163-165 */
    default: return 1;
  }
}
static inline int orc_within(const orc_cropper* c, const double* p) {
  int w = orc_within_impl(c, p);
  return c->invert ? !w : w;
}

/* order-preserving compaction of points (+normals when nrm != NULL) */
ORC_EXPORT size_t orc_crop(const orc_cropper* c, const double* xyz, const double* nrm, size_t n, double* out_xyz, double* out_nrm) {
  size_t m = 0;
  for (size_t i = 0; i < n; i++) {
    if (orc_within(c, xyz + 3 * i)) {
      memcpy(out_xyz + 3 * m, xyz + 3 * i, 24);
      if (nrm && out_nrm) memcpy(out_nrm + 3 * m, nrm + 3 * i, 24);
      m++;
    }
  }
  return m;
}

/* ------------------------------------------------------------------------- */
/*  generic open-addressing voxel hash used by P2 / F1 / F3 restatements      */
/*  (stands in for std::unordered_map<Eigen::Vector3i, ...>; iteration order  */
/*   = first-touch order)                                                     */
/* ------------------------------------------------------------------------- */
typedef struct { int32_t k[3]; int32_t slot; } vh_entry;
typedef struct { vh_entry* e; size_t cap; size_t cnt; } vhash;

static void vh_init(vhash* h, size_t expected) {
  size_t cap = 64; while (cap < 2 * expected + 8) cap <<= 1;
  h->cap = cap; h->cnt = 0;
  h->e = (vh_entry*)malloc(sizeof(vh_entry) * cap);
  for (size_t i = 0; i < cap; i++) h->e[i].slot = -1;
}
static void vh_free(vhash* h) { free(h->e); h->e = NULL; }
static inline uint64_t vh_mix(int32_t x, int32_t y, int32_t z) {
  uint64_t v = (uint64_t)(uint32_t)x * 0x9E3779B97F4A7C15ull;
  v ^= ((uint64_t)(uint32_t)y + 0x7F4A7C15ull) * 0xC2B2AE3D27D4EB4Full;
  v ^= ((uint64_t)(uint32_t)z + 0x165667B1ull) * 0xD6E8FEB86659FD93ull;
  v ^= v >> 29; v *= 0xBF58476D1CE4E5B9ull; v ^= v >> 32;
  return v;
}
/* returns slot id (dense, in first-touch order); *is_new set when inserted */
static int32_t vh_get(vhash* h, int32_t x, int32_t y, int32_t z, int insert, int* is_new) {
  size_t mask = h->cap - 1;
  size_t i = (size_t)vh_mix(x, y, z) & mask;
  for (;;) {
    vh_entry* e = &h->e[i];
    if (e->slot < 0) {
      if (!insert) return -1;
      e->k[0] = x; e->k[1] = y; e->k[2] = z; e->slot = (int32_t)h->cnt++;
      if (is_new) *is_new = 1;
      return e->slot;
    }
    if (e->k[0] == x && e->k[1] == y && e->k[2] == z) { if (is_new) *is_new = 0; return e->slot; }
    i = (i + 1) & mask;
  }
}

/* ------------------------------------------------------------------------- */
/*  P2  voxelize -> [O3D] PointCloud::VoxelDownSample                          */
/*      core/src/helpers.cpp:107-113 ; [O3D] cpp/open3d/geometry/PointCloud.cpp */
/*  key = floor((p - (minBound - v/2)) / v) ; mean of points (+ normals)      */
/*  out_keys (optional, 3 x int32 per voxel) lets tests compare as keyed sets */
/* ------------------------------------------------------------------------- */
ORC_EXPORT size_t orc_voxel_down_sample(const double* xyz, const double* nrm, size_t n, double voxel,
                                        double* out_xyz, double* out_nrm, int32_t* out_keys) {
  if (n == 0) return 0;
  if (voxel <= 0.0) { /* helpers.cpp:108-110 returns the cloud untouched */
    memcpy(out_xyz, xyz, 24 * n);
    if (nrm && out_nrm) memcpy(out_nrm, nrm, 24 * n);
    return n;
  }
  double mn[3] = {xyz[0], xyz[1], xyz[2]};
  for (size_t i = 1; i < n; i++) for (int d = 0; d < 3; d++) if (xyz[3 * i + d] < mn[d]) mn[d] = xyz[3 * i + d];
  double vmin[3];
  for (int d = 0; d < 3; d++) vmin[d] = mn[d] - voxel * 0.5;
  vhash h; vh_init(&h, n);
  double* acc = (double*)calloc(n * 6, sizeof(double));
  int32_t* cnt = (int32_t*)calloc(n, sizeof(int32_t));
  for (size_t i = 0; i < n; i++) {
    int32_t k[3];
    for (int d = 0; d < 3; d++) k[d] = (int32_t)floor((xyz[3 * i + d] - vmin[d]) / voxel);
    int is_new;
    int32_t s = vh_get(&h, k[0], k[1], k[2], 1, &is_new);
    if (is_new && out_keys) { out_keys[3 * s] = k[0]; out_keys[3 * s + 1] = k[1]; out_keys[3 * s + 2] = k[2]; }
    /* AccumulatedPoint::AddPoint */
    acc[6 * s + 0] += xyz[3 * i + 0]; acc[6 * s + 1] += xyz[3 * i + 1]; acc[6 * s + 2] += xyz[3 * i + 2];
    if (nrm) {
      const double* q = nrm + 3 * i;
      if (!isnan(q[0]) && !isnan(q[1]) && !isnan(q[2])) { acc[6 * s + 3] += q[0]; acc[6 * s + 4] += q[1]; acc[6 * s + 5] += q[2]; }
    }
    cnt[s]++;
  }
  size_t m = h.cnt;
  for (size_t s = 0; s < m; s++) {
    double c = (double)cnt[s];
    for (int d = 0; d < 3; d++) out_xyz[3 * s + d] = acc[6 * s + d] / c;
    if (nrm && out_nrm) for (int d = 0; d < 3; d++) out_nrm[3 * s + d] = acc[6 * s + 3 + d] / c;
  }
  free(acc); free(cnt); vh_free(&h);
  return m;
}

/* ------------------------------------------------------------------------- */
/*  P3  estimateNormalsOrCovariancesIfNeeded   core/src/CloudRegistration.cpp:49-56 */
/*      [O3D] EstimateNormals(KDTreeSearchParamHybrid) + NormalizeNormals +   */
/*      OrientNormalsTowardsCameraLocation(0)  (cpp/open3d/geometry/EstimateNormals.cpp, */
/*      PointCloud.cpp, utility/Eigen.h ComputeCovariance)                    */
/* ------------------------------------------------------------------------- */
static void cross3(const double* a, const double* b, double* o) {
  o[0] = a[1] * b[2] - a[2] * b[1]; o[1] = a[2] * b[0] - a[0] * b[2]; o[2] = a[0] * b[1] - a[1] * b[0];
}
static inline double dot3(const double* a, const double* b) { return a[0] * b[0] + a[1] * b[1] + a[2] * b[2]; }

/* A is symmetric, stored full 3x3 row-major */
static void compute_eigenvector0(const double A[9], double eval0, double* out) {
  double row0[3] = {A[0] - eval0, A[1], A[2]};
  double row1[3] = {A[1], A[4] - eval0, A[5]};
  double row2[3] = {A[2], A[5], A[8] - eval0};
  double r0xr1[3], r0xr2[3], r1xr2[3];
  cross3(row0, row1, r0xr1); cross3(row0, row2, r0xr2); cross3(row1, row2, r1xr2);
  double d0 = dot3(r0xr1, r0xr1), d1 = dot3(r0xr2, r0xr2), d2 = dot3(r1xr2, r1xr2);
  double dmax = d0; int imax = 0;
  if (d1 > dmax) { dmax = d1; imax = 1; }
  if (d2 > dmax) { imax = 2; }
  const double* v = imax == 0 ? r0xr1 : (imax == 1 ? r0xr2 : r1xr2);
  double s = sqrt(imax == 0 ? d0 : (imax == 1 ? d1 : d2));
  out[0] = v[0] / s; out[1] = v[1] / s; out[2] = v[2] / s;
}

static void compute_eigenvector1(const double A[9], const double* evec0, double eval1, double* out) {
  double U[3], V[3];
  if (fabs(evec0[0]) > fabs(evec0[1])) {
    double inv = 1 / sqrt(evec0[0] * evec0[0] + evec0[2] * evec0[2]);
    U[0] = -evec0[2] * inv; U[1] = 0; U[2] = evec0[0] * inv;
  } else {
    double inv = 1 / sqrt(evec0[1] * evec0[1] + evec0[2] * evec0[2]);
    U[0] = 0; U[1] = evec0[2] * inv; U[2] = -evec0[1] * inv;
  }
  cross3(evec0, U, V);
  double AU[3] = {A[0] * U[0] + A[1] * U[1] + A[2] * U[2], A[1] * U[0] + A[4] * U[1] + A[5] * U[2], A[2] * U[0] + A[5] * U[1] + A[8] * U[2]};
  double AV[3] = {A[0] * V[0] + A[1] * V[1] + A[2] * V[2], A[1] * V[0] + A[4] * V[1] + A[5] * V[2], A[2] * V[0] + A[5] * V[1] + A[8] * V[2]};
  double m00 = dot3(U, AU) - eval1, m01 = dot3(U, AV), m11 = dot3(V, AV) - eval1;
  double a00 = fabs(m00), a01 = fabs(m01), a11 = fabs(m11);
  if (a00 >= a11) {
    double mx = a00 > a01 ? a00 : a01;
    if (mx > 0) {
      if (a00 >= a01) { m01 /= m00; m00 = 1 / sqrt(1 + m01 * m01); m01 *= m00; }
      else { m00 /= m01; m01 = 1 / sqrt(1 + m00 * m00); m00 *= m01; }
      for (int d = 0; d < 3; d++) out[d] = m01 * U[d] - m00 * V[d];
    } else { out[0] = U[0]; out[1] = U[1]; out[2] = U[2]; }
  } else {
    double mx = a11 > a01 ? a11 : a01;
    if (mx > 0) {
      if (a11 >= a01) { m01 /= m11; m11 = 1 / sqrt(1 + m01 * m01); m01 *= m11; }
      else { m11 /= m01; m01 = 1 / sqrt(1 + m11 * m11); m11 *= m01; }
      for (int d = 0; d < 3; d++) out[d] = m11 * U[d] - m01 * V[d];
    } else { out[0] = U[0]; out[1] = U[1]; out[2] = U[2]; }
  }
}

/* [O3D] FastEigen3x3 (EstimateNormals.cpp): eigenvector of the smallest eigenvalue */
ORC_EXPORT void orc_fast_eigen3x3(const double cov[9], double* out) {
  double A[9]; memcpy(A, cov, sizeof(A));
  double max_coeff = A[0];
  for (int i = 1; i < 9; i++) if (A[i] > max_coeff) max_coeff = A[i];
  if (max_coeff == 0) { out[0] = out[1] = out[2] = 0; return; }
  for (int i = 0; i < 9; i++) A[i] /= max_coeff;
  double norm = A[1] * A[1] + A[2] * A[2] + A[5] * A[5];
  if (norm > 0) {
    double eval[3], evec0[3], evec1[3], evec2[3];
    double q = (A[0] + A[4] + A[8]) / 3;
    double b00 = A[0] - q, b11 = A[4] - q, b22 = A[8] - q;
    double p = sqrt((b00 * b00 + b11 * b11 + b22 * b22 + norm * 2) / 6);
    double c00 = b11 * b22 - A[5] * A[5];
    double c01 = A[1] * b22 - A[5] * A[2];
    double c02 = A[1] * A[5] - b11 * A[2];
    double det = (b00 * c00 - A[1] * c01 + A[2] * c02) / (p * p * p);
    double half_det = det * 0.5;
    half_det = fmin(fmax(half_det, -1.0), 1.0);
    double angle = acos(half_det) / 3.0;
    const double two_thirds_pi = 2.09439510239319549;
    double beta2 = cos(angle) * 2;
    double beta0 = cos(angle + two_thirds_pi) * 2;
    double beta1 = -(beta0 + beta2);
    eval[0] = q + p * beta0; eval[1] = q + p * beta1; eval[2] = q + p * beta2;
    if (half_det >= 0) {
      compute_eigenvector0(A, eval[2], evec2);
      if (eval[2] < eval[0] && eval[2] < eval[1]) { memcpy(out, evec2, 24); return; }
      compute_eigenvector1(A, evec2, eval[1], evec1);
      if (eval[1] < eval[0] && eval[1] < eval[2]) { memcpy(out, evec1, 24); return; }
      cross3(evec1, evec2, evec0);
      memcpy(out, evec0, 24); return;
    } else {
      compute_eigenvector0(A, eval[0], evec0);
      if (eval[0] < eval[1] && eval[0] < eval[2]) { memcpy(out, evec0, 24); return; }
      compute_eigenvector1(A, evec0, eval[1], evec1);
      if (eval[1] < eval[0] && eval[1] < eval[2]) { memcpy(out, evec1, 24); return; }
      cross3(evec0, evec1, evec2);
      memcpy(out, evec2, 24); return;
    }
  } else {
    /* diagonal matrix (A *= max_coeff in the original leaves the ordering unchanged for max_coeff > 0;
       for max_coeff < 0 it flips it, so undo the scaling literally) */
    double a0 = A[0] * max_coeff, a1 = A[4] * max_coeff, a2 = A[8] * max_coeff;
    if (a0 < a1 && a0 < a2) { out[0] = 1; out[1] = 0; out[2] = 0; }
    else if (a1 < a0 && a1 < a2) { out[0] = 0; out[1] = 1; out[2] = 0; }
    else { out[0] = 0; out[1] = 0; out[2] = 1; }
  }
}

/* [O3D] utility::ComputeCovariance: single-pass cumulants, neighbours in the order returned by the search */
static void compute_covariance(const double* pts, const int* idx, int k, double cov[9]) {
  double c[9] = {0};
  for (int j = 0; j < k; j++) {
    const double* p = pts + 3 * idx[j];
    c[0] += p[0]; c[1] += p[1]; c[2] += p[2];
    c[3] += p[0] * p[0]; c[4] += p[0] * p[1]; c[5] += p[0] * p[2];
    c[6] += p[1] * p[1]; c[7] += p[1] * p[2]; c[8] += p[2] * p[2];
  }
  for (int j = 0; j < 9; j++) c[j] /= (double)k;
  cov[0] = c[3] - c[0] * c[0];
  cov[4] = c[6] - c[1] * c[1];
  cov[8] = c[8] - c[2] * c[2];
  cov[1] = cov[3] = c[4] - c[0] * c[1];
  cov[2] = cov[6] = c[5] - c[0] * c[2];
  cov[5] = cov[7] = c[7] - c[1] * c[2];
}

/* full P3: covariances -> normal -> NormalizeNormals -> OrientNormalsTowardsCameraLocation(0,0,0).
 * The cloud is assumed to have no normals/covariances on entry (true at every reference call site
 * on this path: ScanToMapRegistration.cpp:38, Odometry.cpp:28 run it right after voxelize()).
 * out_cov (optional, 9 doubles/pt) exposes the intermediate covariance for tests. */
ORC_EXPORT void orc_estimate_normals(const double* xyz, size_t n, int knn, double radius, double* out_nrm, double* out_cov) {
  kd_tree* t = kd_build(xyz, (int)n);
#pragma omp parallel
  {
    double* d2 = (double*)malloc(sizeof(double) * (size_t)(knn > 0 ? knn : 1));
    int* idx = (int*)malloc(sizeof(int) * (size_t)(knn > 0 ? knn : 1));
#pragma omp for schedule(static)
    for (long i = 0; i < (long)n; i++) {
      double cov[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1};
      int k = kd_search_hybrid(t, xyz + 3 * i, radius, knn, d2, idx);
      if (k >= 3) compute_covariance(xyz, idx, k, cov);
      if (out_cov) memcpy(out_cov + 9 * i, cov, sizeof(cov));
      double nr[3];
      orc_fast_eigen3x3(cov, nr);
      if (sqrt(dot3(nr, nr)) == 0.0) { nr[0] = 0; nr[1] = 0; nr[2] = 1; }
      /* NormalizeNormals: Eigen normalize() leaves a zero vector untouched; NaN -> (0,0,1) */
      double z = dot3(nr, nr);
      if (z > 0) { double s = sqrt(z); nr[0] /= s; nr[1] /= s; nr[2] /= s; }
      if (isnan(nr[0])) { nr[0] = 0; nr[1] = 0; nr[2] = 1; }
      /* OrientNormalsTowardsCameraLocation(camera = 0) */
      double ref[3] = {-xyz[3 * i], -xyz[3 * i + 1], -xyz[3 * i + 2]};
      if (sqrt(dot3(nr, nr)) == 0.0) {
        double rn = sqrt(dot3(ref, ref));
        if (rn == 0.0) { nr[0] = 0; nr[1] = 0; nr[2] = 1; }
        else { nr[0] = ref[0] / rn; nr[1] = ref[1] / rn; nr[2] = ref[2] / rn; }
      } else if (dot3(nr, ref) < 0.0) { nr[0] *= -1.0; nr[1] *= -1.0; nr[2] *= -1.0; }
      out_nrm[3 * i] = nr[0]; out_nrm[3 * i + 1] = nr[1]; out_nrm[3 * i + 2] = nr[2];
    }
    free(d2); free(idx);
  }
  kd_free(t);
}

/* ------------------------------------------------------------------------- */
/*  P4  [O3D] PointCloud::RandomDownSample(ratio)                              */
/*      called at core/src/ScanToMapRegistration.cpp:39, core/src/Odometry.cpp:29 */
/*  Reference: shuffle with mt19937(random_device) and keep floor(ratio*n).    */
/*  Seeded stand-in: keep the floor(ratio*n) points with the smallest          */
/*  (hash(seed,i), i); output keeps the input order.                           */
/* ------------------------------------------------------------------------- */
/* the hash is taken over the BIT PATTERN of the point, not over its index, so that the selected subset does not
 * depend on the (unspecified) order in which the voxel down-sample emitted the points */
ORC_EXPORT uint32_t orc_select_hash(uint32_t seed, const double* p) {
  uint64_t a, b, c;
  memcpy(&a, p, 8); memcpy(&b, p + 1, 8); memcpy(&c, p + 2, 8);
  uint64_t v = a * 0x9E3779B97F4A7C15ull;
  v ^= (b + 0x7F4A7C15F39CC060ull) * 0xC2B2AE3D27D4EB4Full;
  v ^= (c + 0x165667B19E3779F9ull) * 0xD6E8FEB86659FD93ull;
  v += (uint64_t)seed * 0x85EBCA77C2B2AE63ull;
  v ^= v >> 29; v *= 0xBF58476D1CE4E5B9ull; v ^= v >> 32; v *= 0x94D049BB133111EBull; v ^= v >> 29;
  return (uint32_t)(v >> 32);
}
typedef struct { uint32_t h; uint32_t i; } hpair;
static int hpair_cmp(const void* a, const void* b) {
  const hpair* x = (const hpair*)a; const hpair* y = (const hpair*)b;
  if (x->h != y->h) return x->h < y->h ? -1 : 1;
  return x->i < y->i ? -1 : (x->i > y->i ? 1 : 0);
}
ORC_EXPORT size_t orc_random_down_sample(const double* xyz, const double* nrm, size_t n, double ratio, uint32_t seed,
                                         double* out_xyz, double* out_nrm) {
  size_t k = (size_t)((double)n * ratio); /* [O3D]: size_t(points_.size() * sampling_ratio) */
  if (k > n) k = n;
  uint8_t* keep = (uint8_t*)calloc(n ? n : 1, 1);
  if (k == n) memset(keep, 1, n);
  else {
    hpair* hp = (hpair*)malloc(sizeof(hpair) * (n ? n : 1));
    for (size_t i = 0; i < n; i++) { hp[i].h = orc_select_hash(seed, xyz + 3 * i); hp[i].i = (uint32_t)i; }
    qsort(hp, n, sizeof(hpair), hpair_cmp);
    for (size_t j = 0; j < k; j++) keep[hp[j].i] = 1;
    free(hp);
  }
  size_t m = 0;
  for (size_t i = 0; i < n; i++) if (keep[i]) {
    memcpy(out_xyz + 3 * m, xyz + 3 * i, 24);
    if (nrm && out_nrm) memcpy(out_nrm + 3 * m, nrm + 3 * i, 24);
    m++;
  }
  free(keep);
  return m;
}

/* ------------------------------------------------------------------------- */
/*  R1-R5  registerClouds -> [O3D] RegistrationICP + TransformationEstimationPointToPlane */
/*      core/src/CloudRegistration.cpp:44-48 ; [O3D] pipelines/registration/Registration.cpp, */
/*      TransformationEstimation.cpp, utility/Eigen.cpp                        */
/* ------------------------------------------------------------------------- */
typedef struct {
  double T[16];       /* row-major 4x4 */
  double fitness;
  double inlier_rmse;
  int32_t n_corr;
  int32_t iters;      /* number of ComputeTransformation calls executed */
} orc_icp_result;

static void mat4_mul(const double* A, const double* B, double* C) {
  double t[16];
  for (int i = 0; i < 4; i++) for (int j = 0; j < 4; j++) {
    double s = 0; for (int k = 0; k < 4; k++) s += A[4 * i + k] * B[4 * k + j];
    t[4 * i + j] = s;
  }
  memcpy(C, t, sizeof(t));
}
static void mat4_identity(double* T) { memset(T, 0, 128); T[0] = T[5] = T[10] = T[15] = 1.0; }

/* Eigen isIdentity(prec = 1e-12): diagonal ~ 1, off-diagonals much smaller than 1 */
static int mat4_is_identity(const double* T) {
  const double prec = 1e-12;
  for (int i = 0; i < 4; i++) for (int j = 0; j < 4; j++) {
    double v = T[4 * i + j];
    if (i == j) { if (!(fabs(v - 1.0) <= prec * fmin(fabs(v), 1.0))) return 0; }
    else { if (!(fabs(v) <= prec)) return 0; }
  }
  return 1;
}

/* [O3D] PointCloud::Transform -> TransformPoints: p = (T*(p,1)).head3 / w */
static void transform_points(const double* T, double* xyz, size_t n) {
#pragma omp parallel for schedule(static)
  for (long i = 0; i < (long)n; i++) {
    double* p = xyz + 3 * i;
    double x = T[0] * p[0] + T[1] * p[1] + T[2] * p[2] + T[3];
    double y = T[4] * p[0] + T[5] * p[1] + T[6] * p[2] + T[7];
    double z = T[8] * p[0] + T[9] * p[1] + T[10] * p[2] + T[11];
    double w = T[12] * p[0] + T[13] * p[1] + T[14] * p[2] + T[15];
    p[0] = x / w; p[1] = y / w; p[2] = z / w;
  }
}

/* [O3D] GetRegistrationResultAndCorrespondences: SearchHybrid(p, r, 1) per source point */
static void icp_correspondences(const kd_tree* t, const double* src, size_t n_src, double r, int* corr, double* d2out,
                                double* fitness, double* rmse, int* n_corr) {
#pragma omp parallel for schedule(static)
  for (long i = 0; i < (long)n_src; i++) {
    double d2; int idx;
    int k = kd_search_hybrid(t, src + 3 * i, r, 1, &d2, &idx);
    corr[i] = k > 0 ? idx : -1;
    d2out[i] = k > 0 ? d2 : 0.0;
  }
  /* deterministic chunked reduction (reference: per-thread partial sums merged in a critical section) */
  double err2 = 0.0; size_t cnt = 0;
  for (size_t c0 = 0; c0 < n_src; c0 += 1024) {
    double e = 0.0; size_t c1 = c0 + 1024 < n_src ? c0 + 1024 : n_src;
    for (size_t i = c0; i < c1; i++) if (corr[i] >= 0) { e += d2out[i]; cnt++; }
    err2 += e;
  }
  *n_corr = (int)cnt;
  if (cnt == 0) { *fitness = 0.0; *rmse = 0.0; }
  else { *fitness = (double)cnt / (double)n_src; *rmse = sqrt(err2 / (double)cnt); }
}

/* Eigen-style LDLT (symmetric diagonal pivoting on the largest |diagonal|) solve of A x = b, A 6x6 symmetric.
 * [O3D] SolveLinearSystemPSD(JTJ, -JTr) = A.ldlt().solve(b), no det/PSD check on this path. */
ORC_EXPORT void orc_ldlt6_solve(const double* A_in, const double* b_in, double* x) {
  double A[36]; memcpy(A, A_in, sizeof(A));
  int perm[6]; for (int i = 0; i < 6; i++) perm[i] = i;
  /* in-place LDL^T on the lower triangle with symmetric pivoting: P A P^T = L D L^T */
  for (int k = 0; k < 6; k++) {
    int piv = k; double best = fabs(A[7 * k]);
    for (int i = k + 1; i < 6; i++) if (fabs(A[7 * i]) > best) { best = fabs(A[7 * i]); piv = i; }
    if (piv != k) {
      for (int j = 0; j < 6; j++) { double t = A[6 * k + j]; A[6 * k + j] = A[6 * piv + j]; A[6 * piv + j] = t; }
      for (int j = 0; j < 6; j++) { double t = A[6 * j + k]; A[6 * j + k] = A[6 * j + piv]; A[6 * j + piv] = t; }
      int t = perm[k]; perm[k] = perm[piv]; perm[piv] = t;
    }
    double d = A[7 * k];
    if (d != 0.0) {
      for (int i = k + 1; i < 6; i++) A[6 * i + k] /= d;
      for (int i = k + 1; i < 6; i++) for (int j = k + 1; j <= i; j++) {
        A[6 * i + j] -= A[6 * i + k] * d * A[6 * j + k];
        A[6 * j + i] = A[6 * i + j];
      }
    }
  }
  double y[6];
  for (int i = 0; i < 6; i++) y[i] = b_in[perm[i]];
  for (int i = 0; i < 6; i++) for (int j = 0; j < i; j++) y[i] -= A[6 * i + j] * y[j];
  for (int i = 0; i < 6; i++) { double d = A[7 * i]; y[i] = (fabs(d) > 2.2250738585072014e-308) ? y[i] / d : 0.0; } /* Eigen: pseudo-inverse of D */
  for (int i = 5; i >= 0; i--) for (int j = i + 1; j < 6; j++) y[i] -= A[6 * j + i] * y[j];
  for (int i = 0; i < 6; i++) x[perm[i]] = y[i];
}

/* [O3D] TransformVector6dToMatrix4d: R = Rz(x[2]) * Ry(x[1]) * Rx(x[0]), t = x[3..5] */
ORC_EXPORT void orc_vec6_to_mat4(const double* x, double* T) {
  double ca = cos(x[0]), sa = sin(x[0]), cb = cos(x[1]), sb = sin(x[1]), cg = cos(x[2]), sg = sin(x[2]);
  mat4_identity(T);
  T[0] = cg * cb; T[1] = cg * sb * sa - sg * ca; T[2] = cg * sb * ca + sg * sa;
  T[4] = sg * cb; T[5] = sg * sb * sa + cg * ca; T[6] = sg * sb * ca - cg * sa;
  T[8] = -sb;     T[9] = cb * sa;                T[10] = cb * ca;
  T[3] = x[3]; T[7] = x[4]; T[11] = x[5];
}

/* [O3D] TransformationEstimationPointToPlane::ComputeTransformation (L2 loss, w = 1).
 * out_JTJ (36) / out_JTr (6) optional. */
static void p2plane_update(const double* src, const double* tgt, const double* tgt_nrm, const int* corr, size_t n_src,
                           double* update, double* out_JTJ, double* out_JTr) {
  double JTJ[36] = {0}, JTr[6] = {0};
  size_t ncorr = 0;
  for (size_t c0 = 0; c0 < n_src; c0 += 1024) {
    double A[36] = {0}, g[6] = {0};
    size_t c1 = c0 + 1024 < n_src ? c0 + 1024 : n_src;
    for (size_t i = c0; i < c1; i++) {
      int j = corr[i]; if (j < 0) continue;
      ncorr++;
      const double* vs = src + 3 * i; const double* vt = tgt + 3 * j; const double* nt = tgt_nrm + 3 * j;
      double r = (vs[0] - vt[0]) * nt[0] + (vs[1] - vt[1]) * nt[1] + (vs[2] - vt[2]) * nt[2];
      double J[6];
      J[0] = vs[1] * nt[2] - vs[2] * nt[1]; J[1] = vs[2] * nt[0] - vs[0] * nt[2]; J[2] = vs[0] * nt[1] - vs[1] * nt[0];
      J[3] = nt[0]; J[4] = nt[1]; J[5] = nt[2];
      for (int a = 0; a < 6; a++) { for (int b = 0; b < 6; b++) A[6 * a + b] += J[a] * J[b]; g[a] += J[a] * r; }
    }
    for (int a = 0; a < 36; a++) JTJ[a] += A[a];
    for (int a = 0; a < 6; a++) JTr[a] += g[a];
  }
  if (out_JTJ) memcpy(out_JTJ, JTJ, sizeof(JTJ));
  if (out_JTr) memcpy(out_JTr, JTr, sizeof(JTr));
  if (ncorr == 0) { mat4_identity(update); return; }
  double nb[6], x[6];
  for (int a = 0; a < 6; a++) nb[a] = -JTr[a];
  orc_ldlt6_solve(JTJ, nb, x);
  orc_vec6_to_mat4(x, update);
}

/* trace (optional): per evaluation e = 0..iters : fitness, rmse, then JTJ(36)+JTr(6) of the update computed
 * from it  -> 44 doubles per record, trace_cap records max */
ORC_EXPORT int orc_registration_icp_p2plane(const double* src_xyz, size_t n_src, const double* tgt_xyz, const double* tgt_nrm,
                                            size_t n_tgt, double max_corr_dist, const double* init, int max_iter,
                                            double rel_fitness, double rel_rmse, orc_icp_result* out, double* trace,
                                            int trace_cap) {
  if (max_corr_dist <= 0.0) return -1;       /* [O3D] LogError */
  if (!tgt_nrm) return -2;                   /* [O3D] LogError: target needs normals */
  double T[16]; memcpy(T, init, sizeof(T));
  kd_tree* t = kd_build(tgt_xyz, (int)n_tgt); /* rebuilt on every call, like the reference */
  double* pcd = (double*)malloc(24 * (n_src ? n_src : 1));
  memcpy(pcd, src_xyz, 24 * n_src);
  if (!mat4_is_identity(init)) transform_points(init, pcd, n_src);
  int* corr = (int*)malloc(sizeof(int) * (n_src ? n_src : 1));
  double* d2 = (double*)malloc(sizeof(double) * (n_src ? n_src : 1));
  double fit, rmse; int nc;
  icp_correspondences(t, pcd, n_src, max_corr_dist, corr, d2, &fit, &rmse, &nc);
  int it = 0;
  for (int i = 0; i < max_iter; i++) {
    double upd[16], JTJ[36], JTr[6];
    p2plane_update(pcd, tgt_xyz, tgt_nrm, corr, n_src, upd, JTJ, JTr);
    if (trace && i < trace_cap) { trace[44 * i] = fit; trace[44 * i + 1] = rmse; memcpy(trace + 44 * i + 2, JTJ, 288); memcpy(trace + 44 * i + 38, JTr, 48); }
    mat4_mul(upd, T, T);
    transform_points(upd, pcd, n_src);
    double bfit = fit, brmse = rmse;
    icp_correspondences(t, pcd, n_src, max_corr_dist, corr, d2, &fit, &rmse, &nc);
    it = i + 1;
    if (fabs(bfit - fit) < rel_fitness && fabs(brmse - rmse) < rel_rmse) break;
  }
  memcpy(out->T, T, sizeof(T));
  out->fitness = fit; out->inlier_rmse = rmse; out->n_corr = nc; out->iters = it;
  free(pcd); free(corr); free(d2); kd_free(t);
  return 0;
}

/* ------------------------------------------------------------------------- */
/*  R1' point-to-point ICP ("next" row, SURVEY.md 8f rank 3)                     */
/*      RegistrationIcpPointToPoint::registerClouds  core/src/CloudRegistration.cpp:69-75 */
/*      -> [O3D] RegistrationICP(..., TransformationEstimationPointToPoint())  */
/*      ComputeTransformation = Eigen::umeyama(source_mat, target_mat, with_scaling = false) */
/* ------------------------------------------------------------------------- */
/* 3x3 SVD A = U diag(s) V^T by one-sided Jacobi (Hestenes), singular values sorted descending like Eigen's JacobiSVD.
 * Columns of U that belong to a zero singular value are completed to an orthonormal basis. */
ORC_EXPORT void orc_svd3(const double* A, double* U, double* S, double* V) {
  double W[9], Vm[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1};
  memcpy(W, A, sizeof(W));
  for (int sweep = 0; sweep < 60; sweep++) {
    int rotated = 0;
    for (int p = 0; p < 2; p++) for (int q = p + 1; q < 3; q++) {
      double alpha = 0, beta = 0, gamma = 0;
      for (int i = 0; i < 3; i++) { alpha += W[3 * i + p] * W[3 * i + p]; beta += W[3 * i + q] * W[3 * i + q]; gamma += W[3 * i + p] * W[3 * i + q]; }
      if (gamma == 0.0 || fabs(gamma) <= 1e-16 * sqrt(alpha * beta)) continue;
      rotated = 1;
      double zeta = (beta - alpha) / (2.0 * gamma);
      double t = (zeta >= 0 ? 1.0 : -1.0) / (fabs(zeta) + sqrt(1.0 + zeta * zeta));
      double c = 1.0 / sqrt(1.0 + t * t), sn = c * t;
      for (int i = 0; i < 3; i++) {
        double wp = W[3 * i + p], wq = W[3 * i + q];
        W[3 * i + p] = c * wp - sn * wq; W[3 * i + q] = sn * wp + c * wq;
        double vp = Vm[3 * i + p], vq = Vm[3 * i + q];
        Vm[3 * i + p] = c * vp - sn * vq; Vm[3 * i + q] = sn * vp + c * vq;
      }
    }
    if (!rotated) break;
  }
  double sv[3]; int ord[3] = {0, 1, 2};
  for (int j = 0; j < 3; j++) sv[j] = sqrt(W[j] * W[j] + W[3 + j] * W[3 + j] + W[6 + j] * W[6 + j]);
  for (int a = 0; a < 2; a++) for (int b = 0; b < 2 - a; b++) if (sv[ord[b]] < sv[ord[b + 1]]) { int t = ord[b]; ord[b] = ord[b + 1]; ord[b + 1] = t; }
  const double tiny = 1e-300;
  for (int j = 0; j < 3; j++) {
    int o = ord[j];
    S[j] = sv[o];
    for (int i = 0; i < 3; i++) { V[3 * i + j] = Vm[3 * i + o]; U[3 * i + j] = sv[o] > tiny ? W[3 * i + o] / sv[o] : 0.0; }
  }
  /* complete U for vanishing singular values (sorted: they are the trailing columns) */
  if (!(S[0] > tiny)) { double I[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1}; memcpy(U, I, sizeof(I)); return; }
  if (!(S[1] > tiny)) {   /* any unit vector orthogonal to u0 */
    double u0[3] = {U[0], U[3], U[6]};
    int k = fabs(u0[0]) <= fabs(u0[1]) ? (fabs(u0[0]) <= fabs(u0[2]) ? 0 : 2) : (fabs(u0[1]) <= fabs(u0[2]) ? 1 : 2);
    double e[3] = {0, 0, 0}; e[k] = 1.0;
    double d = e[0] * u0[0] + e[1] * u0[1] + e[2] * u0[2];
    double v[3] = {e[0] - d * u0[0], e[1] - d * u0[1], e[2] - d * u0[2]};
    double nv = sqrt(v[0] * v[0] + v[1] * v[1] + v[2] * v[2]);
    U[1] = v[0] / nv; U[4] = v[1] / nv; U[7] = v[2] / nv;
  }
  /* u2 = u0 x u1 also when the third column is rounding noise that is not orthogonal to the others: an exactly zero row of A keeps
     every column of W in a plane, so W's third column can never become orthogonal to the first two (rank-2 sets such as a level
     plane of points) */
  double c[3] = {U[3] * U[7] - U[6] * U[4], U[6] * U[1] - U[0] * U[7], U[0] * U[4] - U[3] * U[1]};
  if (!(fabs(c[0] * U[2] + c[1] * U[5] + c[2] * U[8]) > 0.5)) { U[2] = c[0]; U[5] = c[1]; U[8] = c[2]; }
}

static double det3(const double* M) {
  return M[0] * (M[4] * M[8] - M[5] * M[7]) - M[1] * (M[3] * M[8] - M[5] * M[6]) + M[2] * (M[3] * M[7] - M[4] * M[6]);
}

/* Eigen::umeyama without scaling, from the correspondences (source i -> target corr[i]); two passes like Eigen
 * (means, then the covariance of the demeaned columns) */
static void p2point_update(const double* src, const double* tgt, const int* corr, size_t n_src, double* update) {
  size_t n = 0;
  double ms[3] = {0, 0, 0}, mt[3] = {0, 0, 0};
  for (size_t i = 0; i < n_src; i++) { int j = corr[i]; if (j < 0) continue; n++; for (int a = 0; a < 3; a++) { ms[a] += src[3 * i + a]; mt[a] += tgt[3 * (size_t)j + a]; } }
  if (n == 0) { mat4_identity(update); return; }
  const double one_over_n = 1.0 / (double)n;
  for (int a = 0; a < 3; a++) { ms[a] *= one_over_n; mt[a] *= one_over_n; }
  double sigma[9] = {0};
  for (size_t i = 0; i < n_src; i++) {
    int j = corr[i]; if (j < 0) continue;
    for (int a = 0; a < 3; a++) for (int b = 0; b < 3; b++) sigma[3 * a + b] += (tgt[3 * (size_t)j + a] - mt[a]) * (src[3 * i + b] - ms[b]);
  }
  for (int a = 0; a < 9; a++) sigma[a] *= one_over_n;
  double U[9], S[3], V[9];
  orc_svd3(sigma, U, S, V);
  double sgn = det3(U) * det3(V) < 0 ? -1.0 : 1.0;   /* Eq. (39): S(m-1) = -1 */
  double R[9];
  for (int a = 0; a < 3; a++) for (int b = 0; b < 3; b++) R[3 * a + b] = U[3 * a] * V[3 * b] + U[3 * a + 1] * V[3 * b + 1] + sgn * U[3 * a + 2] * V[3 * b + 2];
  mat4_identity(update);
  for (int a = 0; a < 3; a++) {
    for (int b = 0; b < 3; b++) update[4 * a + b] = R[3 * a + b];
    update[4 * a + 3] = mt[a] - (R[3 * a] * ms[0] + R[3 * a + 1] * ms[1] + R[3 * a + 2] * ms[2]);
  }
}

ORC_EXPORT int orc_registration_icp_p2point(const double* src_xyz, size_t n_src, const double* tgt_xyz, size_t n_tgt, double max_corr_dist,
                                            const double* init, int max_iter, double rel_fitness, double rel_rmse, orc_icp_result* out) {
  if (max_corr_dist <= 0.0) return -1;       /* [O3D] LogError */
  double T[16]; memcpy(T, init, sizeof(T));
  kd_tree* t = kd_build(tgt_xyz, (int)n_tgt);
  double* pcd = (double*)malloc(24 * (n_src ? n_src : 1));
  memcpy(pcd, src_xyz, 24 * n_src);
  if (!mat4_is_identity(init)) transform_points(init, pcd, n_src);
  int* corr = (int*)malloc(sizeof(int) * (n_src ? n_src : 1));
  double* d2 = (double*)malloc(sizeof(double) * (n_src ? n_src : 1));
  double fit, rmse; int nc;
  icp_correspondences(t, pcd, n_src, max_corr_dist, corr, d2, &fit, &rmse, &nc);
  int it = 0;
  for (int i = 0; i < max_iter; i++) {
    double upd[16];
    p2point_update(pcd, tgt_xyz, corr, n_src, upd);
    mat4_mul(upd, T, T);
    transform_points(upd, pcd, n_src);
    double bfit = fit, brmse = rmse;
    icp_correspondences(t, pcd, n_src, max_corr_dist, corr, d2, &fit, &rmse, &nc);
    it = i + 1;
    if (fabs(bfit - fit) < rel_fitness && fabs(brmse - rmse) < rel_rmse) break;
  }
  memcpy(out->T, T, sizeof(T));
  out->fitness = fit; out->inlier_rmse = rmse; out->n_corr = nc; out->iters = it;
  free(pcd); free(corr); free(d2); kd_free(t);
  return 0;
}

/* ------------------------------------------------------------------------- */
/*  R1'' Generalized ICP ("next" row, SURVEY.md 8f rank 3, second half)          */
/*      RegistrationIcpGeneralized::registerClouds  core/src/CloudRegistration.cpp:15-20 */
/*      -> [O3D] RegistrationGeneralizedICP(source, target, r, init, TransformationEstimationForGeneralizedICP(eps = 1e-3)) */
/*      pipelines/registration/GeneralizedICP.cpp: covariances from normals (GetRotationFromE1ToX),  */
/*      per correspondence M = Ct + Cs, W = M^-1/2, rows of W [-skew(vs) | I] and W d, then the     */
/*      same 6x6 solve / update / convergence loop as point-to-plane; the source covariances are   */
/*      rotated with the cloud by every PointCloud::Transform.                                      */
/* ------------------------------------------------------------------------- */
static void mat3_mul(const double* A, const double* B, double* C) {
  double t[9];
  for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++) t[3 * i + j] = A[3 * i] * B[j] + A[3 * i + 1] * B[3 + j] + A[3 * i + 2] * B[6 + j];
  memcpy(C, t, sizeof(t));
}
static void mat3_mul_bt(const double* A, const double* B, double* C) {   /* A * B^T */
  double t[9];
  for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++) t[3 * i + j] = A[3 * i] * B[3 * j] + A[3 * i + 1] * B[3 * j + 1] + A[3 * i + 2] * B[3 * j + 2];
  memcpy(C, t, sizeof(t));
}
/* [O3D] GetRotationFromE1ToX + Rx * diag(eps,1,1) * Rx^T, row-major 3x3 */
ORC_EXPORT void orc_gicp_covariance_from_normal(const double* n, double eps, double* C) {
  const double c = n[0];                                   /* e1 . x */
  double Rx[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1};
  if (!(c < -0.99)) {
    const double v[3] = {0.0, -n[2], n[1]};                /* e1 x x */
    const double sv[9] = {0, -v[2], v[1], v[2], 0, -v[0], -v[1], v[0], 0};
    double sv2[9]; mat3_mul(sv, sv, sv2);
    const double factor = 1 / (1 + c);
    for (int k = 0; k < 9; k++) Rx[k] = (k % 4 == 0 ? 1.0 : 0.0) + sv[k] + sv2[k] * factor;
  }
  const double D[9] = {eps, 0, 0, 0, 1, 0, 0, 0, 1};
  double t[9]; mat3_mul(Rx, D, t); mat3_mul_bt(t, Rx, C);
}
static int inv3(const double* M, double* Mi) {
  const double a = M[0], b = M[1], c = M[2], d = M[3], e = M[4], f = M[5], g = M[6], h = M[7], i = M[8];
  const double det = a * (e * i - f * h) - b * (d * i - f * g) + c * (d * h - e * g);
  const double id = 1.0 / det;
  Mi[0] = (e * i - f * h) * id; Mi[1] = (c * h - b * i) * id; Mi[2] = (b * f - c * e) * id;
  Mi[3] = (f * g - d * i) * id; Mi[4] = (a * i - c * g) * id; Mi[5] = (c * d - a * f) * id;
  Mi[6] = (d * h - e * g) * id; Mi[7] = (b * g - a * h) * id; Mi[8] = (a * e - b * d) * id;
  return det != 0.0;
}
/* J^T J and J^T r of one correspondence with J = W A, r = W d, W = (Ct+Cs)^-1/2, A = [-skew(vs) | I]:
 *   J^T J = A^T M^-1 A,  J^T r = A^T M^-1 d   (W only ever appears squared) */
static void gicp_update(const double* src, const double* src_cov, const double* tgt, const double* tgt_cov, const int* corr, size_t n_src,
                        double* update) {
  double JTJ[36] = {0}, JTr[6] = {0};
  size_t ncorr = 0;
  for (size_t c0 = 0; c0 < n_src; c0 += 1024) {
    double Acc[36] = {0}, g[6] = {0};
    size_t c1 = c0 + 1024 < n_src ? c0 + 1024 : n_src;
    for (size_t i = c0; i < c1; i++) {
      int j = corr[i]; if (j < 0) continue;
      ncorr++;
      const double* vs = src + 3 * i; const double* vt = tgt + 3 * (size_t)j;
      double M[9], Mi[9];
      for (int k = 0; k < 9; k++) M[k] = tgt_cov[9 * (size_t)j + k] + src_cov[9 * i + k];
      inv3(M, Mi);
      const double d[3] = {vs[0] - vt[0], vs[1] - vt[1], vs[2] - vt[2]};
      /* A (3x6) = [-skew(vs) | I] */
      const double A[18] = {0, vs[2], -vs[1], 1, 0, 0, -vs[2], 0, vs[0], 0, 1, 0, vs[1], -vs[0], 0, 0, 0, 1};
      double MA[18];                                       /* M^-1 A */
      for (int r = 0; r < 3; r++) for (int q = 0; q < 6; q++) MA[6 * r + q] = Mi[3 * r] * A[q] + Mi[3 * r + 1] * A[6 + q] + Mi[3 * r + 2] * A[12 + q];
      const double Md[3] = {Mi[0] * d[0] + Mi[1] * d[1] + Mi[2] * d[2], Mi[3] * d[0] + Mi[4] * d[1] + Mi[5] * d[2], Mi[6] * d[0] + Mi[7] * d[1] + Mi[8] * d[2]};
      for (int a = 0; a < 6; a++) {
        for (int b = 0; b < 6; b++) Acc[6 * a + b] += A[a] * MA[b] + A[6 + a] * MA[6 + b] + A[12 + a] * MA[12 + b];
        g[a] += A[a] * Md[0] + A[6 + a] * Md[1] + A[12 + a] * Md[2];
      }
    }
    for (int a = 0; a < 36; a++) JTJ[a] += Acc[a];
    for (int a = 0; a < 6; a++) JTr[a] += g[a];
  }
  if (ncorr == 0) { mat4_identity(update); return; }
  double nb[6], x[6];
  for (int a = 0; a < 6; a++) nb[a] = -JTr[a];
  orc_ldlt6_solve(JTJ, nb, x);
  orc_vec6_to_mat4(x, update);
}
static void transform_covariances(const double* T, double* cov, size_t n) {   /* [O3D] TransformCovariances: R C R^T */
  const double R[9] = {T[0], T[1], T[2], T[4], T[5], T[6], T[8], T[9], T[10]};
  for (size_t i = 0; i < n; i++) { double t[9]; mat3_mul(R, cov + 9 * i, t); mat3_mul_bt(t, R, cov + 9 * i); }
}

ORC_EXPORT int orc_registration_gicp(const double* src_xyz, const double* src_nrm, size_t n_src, const double* tgt_xyz, const double* tgt_nrm,
                                     size_t n_tgt, double max_corr_dist, const double* init, int max_iter, double rel_fitness, double rel_rmse,
                                     double epsilon, orc_icp_result* out) {
  if (max_corr_dist <= 0.0) return -1;
  if (!src_nrm || !tgt_nrm) return -2;   /* this restatement covers the normals -> covariances branch the reference takes */
  double T[16]; memcpy(T, init, sizeof(T));
  double* sc = (double*)malloc(72 * (n_src ? n_src : 1));
  double* tc = (double*)malloc(72 * (n_tgt ? n_tgt : 1));
  for (size_t i = 0; i < n_src; i++) orc_gicp_covariance_from_normal(src_nrm + 3 * i, epsilon, sc + 9 * i);
  for (size_t j = 0; j < n_tgt; j++) orc_gicp_covariance_from_normal(tgt_nrm + 3 * j, epsilon, tc + 9 * j);
  kd_tree* t = kd_build(tgt_xyz, (int)n_tgt);
  double* pcd = (double*)malloc(24 * (n_src ? n_src : 1));
  memcpy(pcd, src_xyz, 24 * n_src);
  if (!mat4_is_identity(init)) { transform_points(init, pcd, n_src); transform_covariances(init, sc, n_src); }
  int* corr = (int*)malloc(sizeof(int) * (n_src ? n_src : 1));
  double* d2 = (double*)malloc(sizeof(double) * (n_src ? n_src : 1));
  double fit, rmse; int nc;
  icp_correspondences(t, pcd, n_src, max_corr_dist, corr, d2, &fit, &rmse, &nc);
  int it = 0;
  for (int i = 0; i < max_iter; i++) {
    double upd[16];
    gicp_update(pcd, sc, tgt_xyz, tc, corr, n_src, upd);
    mat4_mul(upd, T, T);
    transform_points(upd, pcd, n_src);
    transform_covariances(upd, sc, n_src);
    double bfit = fit, brmse = rmse;
    icp_correspondences(t, pcd, n_src, max_corr_dist, corr, d2, &fit, &rmse, &nc);
    it = i + 1;
    if (fabs(bfit - fit) < rel_fitness && fabs(brmse - rmse) < rel_rmse) break;
  }
  memcpy(out->T, T, sizeof(T));
  out->fitness = fit; out->inlier_rmse = rmse; out->n_corr = nc; out->iters = it;
  free(pcd); free(corr); free(d2); free(sc); free(tc); kd_free(t);
  return 0;
}

/* Brute-force single evaluation (for cross-checking the tree): fitness/rmse/JTJ/JTr at transform T */
ORC_EXPORT void orc_icp_evaluate_bruteforce(const double* src_xyz, size_t n_src, const double* tgt_xyz, const double* tgt_nrm,
                                            size_t n_tgt, double r, const double* T, double* fitness, double* rmse,
                                            double* JTJ, double* JTr, int* corr_out) {
  double* pcd = (double*)malloc(24 * (n_src ? n_src : 1));
  memcpy(pcd, src_xyz, 24 * n_src);
  transform_points(T, pcd, n_src);
  int* corr = (int*)malloc(sizeof(int) * (n_src ? n_src : 1));
  double* d2 = (double*)malloc(sizeof(double) * (n_src ? n_src : 1));
  double r2 = r * r;
#pragma omp parallel for schedule(static)
  for (long i = 0; i < (long)n_src; i++) {
    double best = INFINITY; int bj = -1;
    for (size_t j = 0; j < n_tgt; j++) {
      double d = dist2(pcd + 3 * i, tgt_xyz + 3 * j);
      if (d < best) { best = d; bj = (int)j; }
    }
    if (bj >= 0 && best < r2) { corr[i] = bj; d2[i] = best; } else { corr[i] = -1; d2[i] = 0; }
  }
  double err2 = 0; size_t cnt = 0;
  for (size_t c0 = 0; c0 < n_src; c0 += 1024) {
    double e = 0.0; size_t c1 = c0 + 1024 < n_src ? c0 + 1024 : n_src;
    for (size_t i = c0; i < c1; i++) if (corr[i] >= 0) { e += d2[i]; cnt++; }
    err2 += e;
  }
  *fitness = cnt ? (double)cnt / (double)n_src : 0.0;
  *rmse = cnt ? sqrt(err2 / (double)cnt) : 0.0;
  double upd[16];
  p2plane_update(pcd, tgt_xyz, tgt_nrm, corr, n_src, upd, JTJ, JTr);
  if (corr_out) memcpy(corr_out, corr, sizeof(int) * n_src);
  free(pcd); free(corr); free(d2);
}

/* ------------------------------------------------------------------------- */
/*  F0  o3d_slam::transform          core/src/helpers.cpp:273-305              */
/*  Quirk kept literally: when max|T - I| < 1e-4 the output first receives a    */
/*  copy of the whole cloud and then ALSO every transformed point (2n points).  */
/*  out buffers must hold 2n points. Returns the number of points written.     */
/* ------------------------------------------------------------------------- */
ORC_EXPORT size_t orc_transform(const double* T, const double* xyz, const double* nrm, size_t n, double* out_xyz, double* out_nrm) {
  double mx = 0.0;
  for (int i = 0; i < 4; i++) for (int j = 0; j < 4; j++) {
    double v = fabs(T[4 * i + j] - (i == j ? 1.0 : 0.0)); if (v > mx) mx = v;
  }
  size_t m = 0;
  if (mx < 1e-4) {
    memcpy(out_xyz, xyz, 24 * n);
    if (nrm && out_nrm) memcpy(out_nrm, nrm, 24 * n);
    m = n;
  }
  for (size_t i = 0; i < n; i++) {
    const double* p = xyz + 3 * i;
    double x = T[0] * p[0] + T[1] * p[1] + T[2] * p[2] + T[3] * 1.0;
    double y = T[4] * p[0] + T[5] * p[1] + T[6] * p[2] + T[7] * 1.0;
    double z = T[8] * p[0] + T[9] * p[1] + T[10] * p[2] + T[11] * 1.0;
    double w = T[12] * p[0] + T[13] * p[1] + T[14] * p[2] + T[15] * 1.0;
    out_xyz[3 * m] = x / w; out_xyz[3 * m + 1] = y / w; out_xyz[3 * m + 2] = z / w;
    if (nrm && out_nrm) {
      const double* q = nrm + 3 * i;
      out_nrm[3 * m] = T[0] * q[0] + T[1] * q[1] + T[2] * q[2];
      out_nrm[3 * m + 1] = T[4] * q[0] + T[5] * q[1] + T[6] * q[2];
      out_nrm[3 * m + 2] = T[8] * q[0] + T[9] * q[1] + T[10] * q[2];
    }
    m++;
  }
  return m;
}

/* ------------------------------------------------------------------------- */
/*  F1  voxelizeWithinCroppingVolume   core/src/helpers.cpp:115-183            */
/*      (+ AccumulatedPoint :30-70, getVoxelIdx VoxelHashMap.hpp:47-50)        */
/*  Points inside the cropper are bucketed by floor(p * (1/v)) on the           */
/*  global-origin grid; the bucket output is the mean of its members (an old   */
/*  map point counts as ONE member), normals: mean of non-NaN normals then     */
/*  .normalized(); points outside pass through unchanged and come first.       */
/*  out_keys (optional): 3 x int32 per output point; pass-through points get    */
/*  INT32_MIN in all three.                                                    */
/* ------------------------------------------------------------------------- */
ORC_EXPORT size_t orc_voxelize_within_cropping_volume(double voxel, const orc_cropper* c, const double* xyz, const double* nrm,
                                                      size_t n, double* out_xyz, double* out_nrm, int32_t* out_keys) {
  if (voxel <= 0.0) {
    memcpy(out_xyz, xyz, 24 * n);
    if (nrm && out_nrm) memcpy(out_nrm, nrm, 24 * n);
    return n;
  }
  const double inv = 1.0 / voxel;
  vhash h; vh_init(&h, n);
  double* acc = (double*)calloc((n ? n : 1) * 6, sizeof(double));
  int32_t* cnt = (int32_t*)calloc(n ? n : 1, sizeof(int32_t));
  int32_t* keys = (int32_t*)malloc(sizeof(int32_t) * 3 * (n ? n : 1));
  size_t m = 0;
  for (size_t i = 0; i < n; i++) {
    const double* p = xyz + 3 * i;
    if (orc_within(c, p)) {
      int32_t k0 = (int32_t)floor(p[0] * inv), k1 = (int32_t)floor(p[1] * inv), k2 = (int32_t)floor(p[2] * inv);
      int is_new;
      int32_t s = vh_get(&h, k0, k1, k2, 1, &is_new);
      if (is_new) { keys[3 * s] = k0; keys[3 * s + 1] = k1; keys[3 * s + 2] = k2; }
      acc[6 * s] += p[0]; acc[6 * s + 1] += p[1]; acc[6 * s + 2] += p[2];
      if (nrm) {
        const double* q = nrm + 3 * i;
        if (!isnan(q[0]) && !isnan(q[1]) && !isnan(q[2])) { acc[6 * s + 3] += q[0]; acc[6 * s + 4] += q[1]; acc[6 * s + 5] += q[2]; }
      }
      cnt[s]++;
    } else {
      memcpy(out_xyz + 3 * m, p, 24);
      if (nrm && out_nrm) memcpy(out_nrm + 3 * m, nrm + 3 * i, 24);
      if (out_keys) { out_keys[3 * m] = out_keys[3 * m + 1] = out_keys[3 * m + 2] = INT32_MIN; }
      m++;
    }
  }
  for (size_t s = 0; s < h.cnt; s++) {
    double cd = (double)cnt[s];
    for (int d = 0; d < 3; d++) out_xyz[3 * m + d] = acc[6 * s + d] / cd;
    if (nrm && out_nrm) {
      double a[3] = {acc[6 * s + 3] / cd, acc[6 * s + 4] / cd, acc[6 * s + 5] / cd};
      double z = dot3(a, a);
      if (z > 0) { double sn = sqrt(z); a[0] /= sn; a[1] /= sn; a[2] /= sn; } /* Eigen normalized() */
      out_nrm[3 * m] = a[0]; out_nrm[3 * m + 1] = a[1]; out_nrm[3 * m + 2] = a[2];
    }
    if (out_keys) { out_keys[3 * m] = keys[3 * s]; out_keys[3 * m + 1] = keys[3 * s + 1]; out_keys[3 * m + 2] = keys[3 * s + 2]; }
    m++;
  }
  free(acc); free(cnt); free(keys); vh_free(&h);
  return m;
}

/* Submap::insertScan, sparse map, no carving   core/src/Submap.cpp:39-75
 * map (n_map points + normals) is updated in place into out_* (capacity >= n_map + 2*n_scan). */
ORC_EXPORT size_t orc_submap_insert_scan(const double* map_xyz, const double* map_nrm, size_t n_map, const double* scan_xyz,
                                         const double* scan_nrm, size_t n_scan, const double* T, double map_voxel,
                                         const orc_cropper* map_builder_cropper_at_sensor, double* out_xyz, double* out_nrm,
                                         int32_t* out_keys) {
  if (n_scan == 0) { /* Submap.cpp:41-43 */
    memcpy(out_xyz, map_xyz, 24 * n_map); memcpy(out_nrm, map_nrm, 24 * n_map); return n_map;
  }
  size_t cap = n_map + 2 * n_scan;
  double* cat_xyz = (double*)malloc(24 * cap);
  double* cat_nrm = (double*)malloc(24 * cap);
  memcpy(cat_xyz, map_xyz, 24 * n_map); memcpy(cat_nrm, map_nrm, 24 * n_map);
  size_t nt = orc_transform(T, scan_xyz, scan_nrm, n_scan, cat_xyz + 3 * n_map, cat_nrm + 3 * n_map); /* :54, :70 */
  orc_cropper c = *map_builder_cropper_at_sensor;
  c.center[0] = T[3]; c.center[1] = T[7]; c.center[2] = T[11]; /* :71 setPose(mapToRangeSensor) */
  size_t m = orc_voxelize_within_cropping_volume(map_voxel, &c, cat_xyz, cat_nrm, n_map + nt, out_xyz, out_nrm, out_keys); /* :72 */
  free(cat_xyz); free(cat_nrm);
  return m;
}

/* ------------------------------------------------------------------------- */
/*  F3  VoxelizedPointCloud (dense map)   core/src/Voxel.cpp:18-115            */
/*  running sum of positions / normals and a count per voxel; key =            */
/*  floor(p * (1/v)) (VoxelHashMap.hpp:47-50 via getKey :124)                  */
/* ------------------------------------------------------------------------- */
typedef struct {
  vhash h;
  double inv;
  double* sum;     /* 6 per voxel: position sum, normal sum */
  int32_t* cnt;
  int32_t* keys;
  size_t cap;
  int has_normals;
} orc_dense;

ORC_EXPORT void* orc_dense_create(double voxel, size_t max_voxels) {
  orc_dense* d = (orc_dense*)calloc(1, sizeof(orc_dense));
  vh_init(&d->h, max_voxels);
  d->inv = 1.0 / voxel; d->cap = max_voxels;
  d->sum = (double*)calloc(max_voxels * 6, sizeof(double));
  d->cnt = (int32_t*)calloc(max_voxels, sizeof(int32_t));
  d->keys = (int32_t*)calloc(max_voxels * 3, sizeof(int32_t));
  return d;
}
ORC_EXPORT void orc_dense_destroy(void* p) {
  orc_dense* d = (orc_dense*)p; if (!d) return;
  vh_free(&d->h); free(d->sum); free(d->cnt); free(d->keys); free(d);
}
/* VoxelizedPointCloud::insert  Voxel.cpp:66-88 ; returns -1 when capacity would be exceeded */
ORC_EXPORT int orc_dense_insert(void* p, const double* xyz, const double* nrm, size_t n) {
  orc_dense* d = (orc_dense*)p;
  for (size_t i = 0; i < n; i++) {
    const double* q = xyz + 3 * i;
    int32_t k0 = (int32_t)floor(q[0] * d->inv), k1 = (int32_t)floor(q[1] * d->inv), k2 = (int32_t)floor(q[2] * d->inv);
    if (d->h.cnt >= d->cap && vh_get(&d->h, k0, k1, k2, 0, NULL) < 0) return -1;
    int is_new;
    int32_t s = vh_get(&d->h, k0, k1, k2, 1, &is_new);
    if (is_new) { d->keys[3 * s] = k0; d->keys[3 * s + 1] = k1; d->keys[3 * s + 2] = k2; }
    d->sum[6 * s] += q[0]; d->sum[6 * s + 1] += q[1]; d->sum[6 * s + 2] += q[2];
    d->cnt[s]++;
    if (nrm) { d->sum[6 * s + 3] += nrm[3 * i]; d->sum[6 * s + 4] += nrm[3 * i + 1]; d->sum[6 * s + 5] += nrm[3 * i + 2]; d->has_normals = 1; }
  }
  return 0;
}
/* VoxelizedPointCloud::toPointCloud  Voxel.cpp:90-115 */
ORC_EXPORT size_t orc_dense_to_cloud(void* p, double* out_xyz, double* out_nrm, int32_t* out_keys) {
  orc_dense* d = (orc_dense*)p;
  size_t m = 0;
  for (size_t s = 0; s < d->h.cnt; s++) {
    if (d->cnt[s] <= 0) continue;
    double c = (double)d->cnt[s];
    for (int k = 0; k < 3; k++) out_xyz[3 * m + k] = d->sum[6 * s + k] / c;
    if (out_nrm) for (int k = 0; k < 3; k++) out_nrm[3 * m + k] = d->has_normals ? d->sum[6 * s + 3 + k] / c : 0.0;
    if (out_keys) { out_keys[3 * m] = d->keys[3 * s]; out_keys[3 * m + 1] = d->keys[3 * s + 1]; out_keys[3 * m + 2] = d->keys[3 * s + 2]; }
    m++;
  }
  return m;
}

/* C2  space carving of the DENSE map ("next" row, SURVEY.md 8f rank 1, second half)
 *     Submap::carve(scan, sensorPosition, param, VoxelizedPointCloud*)  core/src/Submap.cpp:125-136
 *     removeDuplicatePointsWithinSameVoxels  core/src/Voxel.cpp:162-192 ; getKeysOfCarvedPoints  core/src/helpers.cpp:347-377
 *     getVoxelsWithinPointNeighborhood  core/src/VoxelHashMap.cpp:13-45 (keys by DIVISION: getVoxelIdx(p, voxelSize))
 *     `scan` is used in whatever frame the caller hands over (the reference passes the raw scan with the map-frame
 *     sensor position, core/src/Submap.cpp:88).  Returns the number of voxels removed. */
ORC_EXPORT size_t orc_dense_carve(void* pd, const double* scan, size_t n, const double* sensor, double voxel, double radius,
                                  double truncation, double max_len) {
  orc_dense* d = (orc_dense*)pd;
  /* removeDuplicatePointsWithinSameVoxels: the first point of every voxel (key by multiplication with 1/voxel) */
  vhash seen; vh_init(&seen, n);
  uint8_t* first = (uint8_t*)calloc(n ? n : 1, 1);
  const double inv = 1.0 / voxel;
  for (size_t i = 0; i < n; i++) {
    int is_new = 0;
    vh_get(&seen, (int32_t)floor(scan[3 * i] * inv), (int32_t)floor(scan[3 * i + 1] * inv), (int32_t)floor(scan[3 * i + 2] * inv), 1, &is_new);
    first[i] = (uint8_t)is_new;
  }
  vh_free(&seen);
  uint8_t* rm = (uint8_t*)calloc(d->h.cnt ? d->h.cnt : 1, 1);
  const double step = 2.0 * radius;
  /* the reference marches the rays under "#pragma omp parallel for schedule(static)" (helpers.cpp:352); here every hit is
   * an idempotent byte store into rm[], so no critical section is needed and the result does not depend on the schedule */
#pragma omp parallel for schedule(dynamic, 256)
  for (size_t i = 0; i < n; i++) {
    if (!first[i]) continue;
    const double* p = scan + 3 * i;
    const double dx = p[0] - sensor[0], dy = p[1] - sensor[1], dz = p[2] - sensor[2];
    const double length = sqrt(dx * dx + dy * dy + dz * dz);
    const double dir[3] = {dx / length, dy / length, dz / length};
    double mp = length - truncation;
    if (max_len < mp) mp = max_len;
    if (step > mp) mp = step;
    if (!(mp == mp)) continue;
    double distance = 0.0;
    while (distance < mp) {
      const double c[3] = {distance * dir[0] + sensor[0], distance * dir[1] + sensor[1], distance * dir[2] + sensor[2]};
      const int32_t ck[3] = {(int32_t)floor(c[0] / voxel), (int32_t)floor(c[1] / voxel), (int32_t)floor(c[2] / voxel)};
      int center_added = 0;
      if (radius <= 0.0) {
        int32_t s0 = vh_get(&d->h, ck[0], ck[1], ck[2], 0, NULL);
        if (s0 >= 0 && d->cnt[s0] > 0) rm[s0] = 1;
        center_added = 1;
      } else {
        for (double ox = -radius; ox <= radius; ox += voxel)
          for (double oy = -radius; oy <= radius; oy += voxel)
            for (double oz = -radius; oz <= radius; oz += voxel) {
              const double t[3] = {c[0] + ox, c[1] + oy, c[2] + oz};
              const int32_t k[3] = {(int32_t)floor(t[0] / voxel), (int32_t)floor(t[1] / voxel), (int32_t)floor(t[2] / voxel)};
              const double e[3] = {t[0] - ((double)k[0] * voxel + voxel * 0.5), t[1] - ((double)k[1] * voxel + voxel * 0.5),
                                   t[2] - ((double)k[2] * voxel + voxel * 0.5)};
              if (sqrt(e[0] * e[0] + e[1] * e[1] + e[2] * e[2]) <= radius) {
                int32_t s0 = vh_get(&d->h, k[0], k[1], k[2], 0, NULL);
                if (s0 >= 0 && d->cnt[s0] > 0) rm[s0] = 1;
                if (k[0] == ck[0] && k[1] == ck[1] && k[2] == ck[2]) center_added = 1;
              }
            }
      }
      if (!center_added) {
        int32_t s0 = vh_get(&d->h, ck[0], ck[1], ck[2], 0, NULL);
        if (s0 >= 0 && d->cnt[s0] > 0) rm[s0] = 1;
      }
      distance += step;
    }
  }
  size_t removed = 0;
  for (size_t s0 = 0; s0 < d->h.cnt; s0++) if (rm[s0]) { d->cnt[s0] = 0; for (int k = 0; k < 6; k++) d->sum[6 * s0 + k] = 0.0; removed++; }   /* removeKey */
  free(first); free(rm);
  return removed;
}

/* ------------------------------------------------------------------------- */
/*  S1  ScanToMapIcp::preprocess + processForScanMatchingAndMerging            */
/*      core/src/ScanToMapRegistration.cpp:35-54 (also Odometry.cpp:25-30)     */
/*  crop(mapBuilder cropper @ identity) -> voxelize -> normals -> random down   */
/*  sample = merge_ ; crop(scanMatcher cropper @ identity) of merge_ = match_   */
/*  All out buffers need capacity n.  Returns 0, or -1 when either is empty.    */
/* ------------------------------------------------------------------------- */
ORC_EXPORT int orc_process_scan(const double* raw_xyz, size_t n, const orc_cropper* map_builder_cropper,
                                const orc_cropper* scan_matcher_cropper, double voxel, int knn, double knn_radius, double ratio,
                                uint32_t seed, double* merge_xyz, double* merge_nrm, size_t* n_merge, double* match_xyz,
                                double* match_nrm, size_t* n_match) {
  double* a = (double*)malloc(24 * (n ? n : 1));
  double* b = (double*)malloc(24 * (n ? n : 1));
  double* bn = (double*)malloc(24 * (n ? n : 1));
  orc_cropper c0 = *map_builder_cropper; c0.center[0] = c0.center[1] = c0.center[2] = 0.0;
  size_t m = orc_crop(&c0, raw_xyz, NULL, n, a, NULL);
  m = orc_voxel_down_sample(a, NULL, m, voxel, b, NULL, NULL);
  if (m > 0) orc_estimate_normals(b, m, knn, knn_radius, bn, NULL);
  size_t k = orc_random_down_sample(b, bn, m, ratio, seed, merge_xyz, merge_nrm);
  *n_merge = k;
  orc_cropper c1 = *scan_matcher_cropper; c1.center[0] = c1.center[1] = c1.center[2] = 0.0;
  *n_match = orc_crop(&c1, merge_xyz, merge_nrm, k, match_xyz, match_nrm);
  free(a); free(b); free(bn);
  return (*n_merge > 0 && *n_match > 0) ? 0 : -1;
}

/* ------------------------------------------------------------------------- */
/*  C1  space carving of the sparse map ("next" row, SURVEY.md 8f rank 1)       */
/*      Submap::carve  core/src/Submap.cpp:109-123                             */
/*      getIdxsOfCarvedPoints  core/src/helpers.cpp:235-271                    */
/*      VoxelMap::insertCloud / getIndicesInVoxel  core/src/Voxel.cpp:123-149  */
/*  scan_xyz: the raw scan ALREADY in the map frame (carve() transforms it);   */
/*  only the map points inside `cropper` are candidates (getIndicesWithinVolume)*/
/*  removed[i] = 1 for every map point hit by a ray that is not (nearly)        */
/*  parallel to its surface.  Returns the number of removed points.             */
/* ------------------------------------------------------------------------- */
typedef struct {
  double voxel_size, max_raytracing_length, truncation_distance, min_dot_product_with_normal;
} orc_carving_params;

ORC_EXPORT size_t orc_carve(const double* map_xyz, const double* map_nrm, size_t n_map, const double* scan_xyz, size_t n_scan,
                            const double* sensor, const orc_cropper* cropper, const orc_carving_params* prm, uint8_t* removed) {
  memset(removed, 0, n_map);
  if (n_map == 0) return 0;
  const double inv = 1.0 / prm->voxel_size;   /* VoxelHashMap.hpp:43-45 fromVoxelSize */
  /* voxel -> chained list of the map indices inside the cropper */
  vhash h; vh_init(&h, n_map);
  int32_t* head = (int32_t*)malloc(sizeof(int32_t) * (n_map + 1));
  int32_t* next = (int32_t*)malloc(sizeof(int32_t) * (n_map + 1));
  for (size_t i = 0; i < n_map; i++) {
    next[i] = -1;
    if (!orc_within(cropper, map_xyz + 3 * i)) continue;
    const double* p = map_xyz + 3 * i;
    int is_new = 0;
    int32_t slot = vh_get(&h, (int32_t)floor(p[0] * inv), (int32_t)floor(p[1] * inv), (int32_t)floor(p[2] * inv), 1, &is_new);
    if (is_new) head[slot] = -1;
    next[i] = head[slot]; head[slot] = (int32_t)i;
  }
  const double step = prm->voxel_size;
#pragma omp parallel for schedule(static)
  for (size_t i = 0; i < n_scan; i++) {
    const double* p = scan_xyz + 3 * i;
    const double dx = p[0] - sensor[0], dy = p[1] - sensor[1], dz = p[2] - sensor[2];
    const double length = sqrt(dx * dx + dy * dy + dz * dz);
    const double dir[3] = {dx / length, dy / length, dz / length};
    double mp = length - prm->truncation_distance;
    if (prm->max_raytracing_length < mp) mp = prm->max_raytracing_length;       /* std::min */
    if (prm->voxel_size > mp) mp = prm->voxel_size;                              /* std::max */
    if (!(mp == mp)) continue;                                                   /* NaN ray: the while condition is false */
    double distance = 0.0;
    while (distance < mp) {
      const double cx = distance * dir[0] + sensor[0], cy = distance * dir[1] + sensor[1], cz = distance * dir[2] + sensor[2];
      int32_t slot = vh_get(&h, (int32_t)floor(cx * inv), (int32_t)floor(cy * inv), (int32_t)floor(cz * inv), 0, NULL);
      if (slot >= 0) {
        for (int32_t id = head[slot]; id >= 0; id = next[id]) {
          int rm = 1;
          if (map_nrm) {
            const double* n = map_nrm + 3 * (size_t)id;
            double nn = sqrt(n[0] * n[0] + n[1] * n[1] + n[2] * n[2]);
            double nx = n[0], ny = n[1], nz = n[2];
            if (nn > 0.0) { nx /= nn; ny /= nn; nz /= nn; }                      /* Eigen normalized(): unchanged when the norm is 0 */
            rm = fabs(dir[0] * nx + dir[1] * ny + dir[2] * nz) > prm->min_dot_product_with_normal;
          }
          if (rm) removed[id] = 1;                                               /* set insert: idempotent */
        }
      }
      distance += step;
    }
  }
  vh_free(&h); free(head); free(next);
  size_t cnt = 0;
  for (size_t i = 0; i < n_map; i++) cnt += removed[i];
  return cnt;
}

/* ------------------------------------------------------------------------- */
/*  L1  overlap selection + information matrix around the loop-closure ICP      */
/*      ("next" row, SURVEY.md 8f rank 2)                                       */
/*      computeIndicesOfOverlappingPoints  core/src/helpers.cpp:307-332         */
/*      [O3D] GetInformationMatrixFromPointClouds (core/src/PlaceRecognition.cpp:148, */
/*      core/src/constraint_builders.cpp:71)                                    */
/* ------------------------------------------------------------------------- */
/* flags (0/1) per source / target point: the point lies in a voxel (key = floor(p * (1/voxel)), source transformed by T
 * like [O3D] PointCloud::Transform) that holds >= min_pts source AND >= min_pts target points.  The reference returns
 * index lists in hash-map order; callers only use them through SelectByIndex, so the sets are what matters. */
ORC_EXPORT void orc_overlap_flags(const double* src, size_t n_src, const double* tgt, size_t n_tgt, const double* T, double voxel,
                                  size_t min_pts, uint8_t* src_flag, uint8_t* tgt_flag) {
  const double inv = 1.0 / voxel;
  double* st = (double*)malloc(24 * (n_src ? n_src : 1));
  memcpy(st, src, 24 * n_src);
  transform_points(T, st, n_src);   /* sourceTransformed.Transform(sourceToTarget.matrix()) -- unconditional here */
  vhash h; vh_init(&h, n_src + n_tgt);
  int32_t* cs = (int32_t*)calloc(n_src + n_tgt + 1, sizeof(int32_t));
  int32_t* ct = (int32_t*)calloc(n_src + n_tgt + 1, sizeof(int32_t));
  int32_t* ss = (int32_t*)malloc(sizeof(int32_t) * (n_src ? n_src : 1));
  int32_t* ts = (int32_t*)malloc(sizeof(int32_t) * (n_tgt ? n_tgt : 1));
  for (size_t j = 0; j < n_tgt; j++) {
    const double* p = tgt + 3 * j;
    ts[j] = vh_get(&h, (int32_t)floor(p[0] * inv), (int32_t)floor(p[1] * inv), (int32_t)floor(p[2] * inv), 1, NULL);
    ct[ts[j]]++;
  }
  for (size_t i = 0; i < n_src; i++) {
    const double* p = st + 3 * i;
    ss[i] = vh_get(&h, (int32_t)floor(p[0] * inv), (int32_t)floor(p[1] * inv), (int32_t)floor(p[2] * inv), 1, NULL);
    cs[ss[i]]++;
  }
  for (size_t i = 0; i < n_src; i++) src_flag[i] = (size_t)cs[ss[i]] >= min_pts && (size_t)ct[ss[i]] >= min_pts;
  for (size_t j = 0; j < n_tgt; j++) tgt_flag[j] = (size_t)cs[ts[j]] >= min_pts && (size_t)ct[ts[j]] >= min_pts;
  vh_free(&h); free(cs); free(ct); free(ss); free(ts); free(st);
}

/* [O3D] GetInformationMatrixFromPointClouds(source, target, max_correspondence_distance, transformation): 6x6 row-major */
ORC_EXPORT int orc_information_matrix(const double* src, size_t n_src, const double* tgt, size_t n_tgt, double max_corr_dist,
                                      const double* T, double* info36) {
  if (max_corr_dist <= 0.0) return -1;
  double* pcd = (double*)malloc(24 * (n_src ? n_src : 1));
  memcpy(pcd, src, 24 * n_src);
  if (!mat4_is_identity(T)) transform_points(T, pcd, n_src);
  kd_tree* t = kd_build(tgt, (int)n_tgt);
  int* corr = (int*)malloc(sizeof(int) * (n_src ? n_src : 1));
  double* d2 = (double*)malloc(sizeof(double) * (n_src ? n_src : 1));
  double fit, rmse; int nc;
  icp_correspondences(t, pcd, n_src, max_corr_dist, corr, d2, &fit, &rmse, &nc);
  double G[36] = {0};
  for (size_t i = 0; i < n_src; i++) {
    int j = corr[i]; if (j < 0) continue;
    const double x = tgt[3 * (size_t)j], y = tgt[3 * (size_t)j + 1], z = tgt[3 * (size_t)j + 2];
    const double r[3][6] = {{0, z, -y, 1, 0, 0}, {-z, 0, x, 0, 1, 0}, {y, -x, 0, 0, 0, 1}};
    for (int k = 0; k < 3; k++) for (int a = 0; a < 6; a++) for (int b = 0; b < 6; b++) G[6 * a + b] += r[k][a] * r[k][b];
  }
  memcpy(info36, G, sizeof(G));
  free(pcd); free(corr); free(d2); kd_free(t);
  return 0;
}

/* ------------------------------------------------------------------------- */
/*  D1  constant-velocity de-skew ("next" row, SURVEY.md 8f rank 4)             */
/*      ConstantVelocityMotionCompensation::undistortInputPointCloud / computePhase */
/*      core/src/MotionCompensation.cpp:64-139 ; fromRPY core/src/math.cpp:32-37 */
/*      makeTransform(xyz, q) * p  =  R(q) p + xyz  (Eigen toRotationMatrix)     */
/* ------------------------------------------------------------------------- */
#ifndef M_PI
#define M_PI 3.14159265358979323846
#endif
static void quat_mul(const double* a, const double* b, double* o) {   /* (w,x,y,z), Eigen's product */
  o[0] = a[0] * b[0] - a[1] * b[1] - a[2] * b[2] - a[3] * b[3];
  o[1] = a[0] * b[1] + a[1] * b[0] + a[2] * b[3] - a[3] * b[2];
  o[2] = a[0] * b[2] + a[2] * b[0] + a[3] * b[1] - a[1] * b[3];
  o[3] = a[0] * b[3] + a[3] * b[0] + a[1] * b[2] - a[2] * b[1];
}
ORC_EXPORT double orc_compute_phase(double x, double y, int spinning_clockwise) {
  const double angle = atan2(y, x);
  const double wrapped = angle < 0.0 ? (angle + 2.0 * M_PI) : angle;
  if (wrapped == 0.0) return 0.0;
  return spinning_clockwise ? 1.0 - wrapped / (2.0 * M_PI) : wrapped / (2.0 * M_PI);
}
ORC_EXPORT void orc_undistort(const double* xyz, size_t n, const double* lin_vel, const double* ang_vel_rpy, double scan_duration,
                              int spinning_clockwise, double* out) {
#pragma omp parallel for schedule(static)
  for (long i = 0; i < (long)n; i++) {
    const double* p = xyz + 3 * i;
    const double phase = orc_compute_phase(p[0], p[1], spinning_clockwise);
    const double s = phase * scan_duration;
    const double t[3] = {s * lin_vel[0], s * lin_vel[1], s * lin_vel[2]};
    const double r = s * ang_vel_rpy[0], pi = s * ang_vel_rpy[1], yw = s * ang_vel_rpy[2];
    const double qx[4] = {cos(0.5 * r), sin(0.5 * r), 0, 0}, qy[4] = {cos(0.5 * pi), 0, sin(0.5 * pi), 0}, qz[4] = {cos(0.5 * yw), 0, 0, sin(0.5 * yw)};
    double qzy[4], q[4];
    quat_mul(qz, qy, qzy); quat_mul(qzy, qx, q);                 /* yaw * pitch * roll */
    const double n2 = q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3];
    if (n2 > 0.0) { const double nn = sqrt(n2); for (int k = 0; k < 4; k++) q[k] /= nn; }   /* .normalized() */
    const double w = q[0], x = q[1], y = q[2], z = q[3];
    const double tx = 2 * x, ty = 2 * y, tz = 2 * z, twx = tx * w, twy = ty * w, twz = tz * w, txx = tx * x, txy = ty * x, txz = tz * x,
                 tyy = ty * y, tyz = tz * y, tzz = tz * z;
    const double R[9] = {1 - (tyy + tzz), txy - twz, txz + twy, txy + twz, 1 - (txx + tzz), tyz - twx, txz - twy, tyz + twx, 1 - (txx + tyy)};
    for (int a = 0; a < 3; a++) out[3 * i + a] = (R[3 * a] * p[0] + R[3 * a + 1] * p[1] + R[3 * a + 2] * p[2]) + t[a];
  }
}

/* ------------------------------------------------------------------------- */
/*  Submap::transform  core/src/Submap.cpp:94-107 (loop-closure correction of a submap)   */
/*  mapCloud_.Transform(mat) = [O3D] PointCloud::Transform: TransformPoints (T p / w),     */
/*  TransformNormals (R n) -- no duplication quirk here; denseMap_.transform(T) =          */
/*  VoxelizedPointCloud::transform (core/src/Voxel.cpp:49-64): the affine map is applied   */
/*  to the SUMS and the keys stay (kept as it is).                                         */
/* ------------------------------------------------------------------------- */
ORC_EXPORT void orc_pointcloud_transform(const double* T, double* xyz, double* nrm, size_t n) {
  transform_points(T, xyz, n);
  if (nrm) for (size_t i = 0; i < n; i++) {
    double* v = nrm + 3 * i;
    const double a = T[0] * v[0] + T[1] * v[1] + T[2] * v[2], b = T[4] * v[0] + T[5] * v[1] + T[6] * v[2], c = T[8] * v[0] + T[9] * v[1] + T[10] * v[2];
    v[0] = a; v[1] = b; v[2] = c;
  }
}
ORC_EXPORT void orc_dense_transform(void* pd, const double* T) {
  orc_dense* d = (orc_dense*)pd;
  for (size_t s0 = 0; s0 < d->h.cnt; s0++) {
    if (d->cnt[s0] <= 0) continue;
    double* v = d->sum + 6 * s0;
    const double a = (T[0] * v[0] + T[1] * v[1] + T[2] * v[2]) + T[3], b = (T[4] * v[0] + T[5] * v[1] + T[6] * v[2]) + T[7],
                 c = (T[8] * v[0] + T[9] * v[1] + T[10] * v[2]) + T[11];
    v[0] = a; v[1] = b; v[2] = c;
  }
}

ORC_EXPORT int orc_num_threads(void) {
#ifdef _OPENMP
  return omp_get_max_threads();
#else
  return 1;
#endif
}
