// odometry.cu -- LidarOdometry (core/src/Odometry.cpp:19-110) with its TransformInterpolationBuffer (TransformInterpolationBuffer.cpp,
// Transform.cpp:16-41) on the device, and the combined per-scan step odometry -> Mapper::addRangeMeasurement (Mapper.cpp:101-181)
// whose prediction is read from that buffer on the device.  Every decision is taken by single-CTA kernels of the chain; the host only
// checks arguments, keeps the timestamp order and enqueues.
#include <map>

#include "common.cuh"

using namespace b2s;

namespace b2s {

// device-resident state of one odometry object
struct OdoState {
  double cum[16];             // odomToRangeSensorCumulative_
  double init_T[16];          // initialTransform_
  long long t_cur;            // timestamp of the step in flight (from the host ring)
  long long t_last;           // the mapper's lastMeasurementTimestamp_ (Time() = 0 until a scan is accepted)
  int32_t init_pending;       // isInitialTransformSet_
  int32_t step;               // device step counter: index into the host ring
  int32_t slot;               // result slot of the step in flight
  int32_t keep;               // cloudPrev_ = pre in this step
  int32_t head, count;        // buffer ring: physical index of the earliest entry, entries held
  int32_t odom_used;          // the step's prediction came from the buffer
  int32_t pad;
  int32_t map_head, map_count;   // the mapper's mapToRangeSensorBuffer_ ring (map_t / map_T), same layout
};

struct OdoStepInput {         // what the host hands each step (pinned, device-mapped ring of 64)
  long long t;
  int32_t slot, pad;
};

struct Mat16 { double v[16]; };

constexpr int ODO_RING = 64;

}  // namespace b2s

struct b2s_odometry {
  b2s_handle* h = nullptr;
  int device = 0;
  b2s_odometry_params params;
  unsigned long long params_gen = 1;   // bumped by b2s_odometry_set_params: the captured combined graphs bake the parameters in
  size_t capacity = 0;
  std::unique_ptr<b2s_cloud> prev;     // cloudPrev_ (fixed capacity: the keep copy writes into it from the device)
  std::unique_ptr<b2s_cloud> pre;      // the pre-processed scan of the step in flight
  std::unique_ptr<b2s_cloud> scratch;  // its voxelized cloud
  std::unique_ptr<b2s_cloud> input;    // upload target of b2s_slam_step_host_async outside graph mode
  std::unique_ptr<b2s_cloud> staging;  // graph mode: the fixed-capacity input cloud every scan is uploaded into
  b2s::GridIndex grid;                 // target index of the registration (the current scan, rebuilt every step)
  b2s::DevBuf state;                   // OdoState
  b2s::DevBuf ring_t, ring_T;          // odomToRangeSensorBuffer_: buffer_size x (int64 time, 4x4)
  b2s::DevBuf map_t, map_T;            // the mapper's mapToRangeSensorBuffer_: buffer_size x (int64 time, 4x4)
  b2s_motion_compensation_params mc;   // de-skew of both inputs (b2s_odometry_set_motion_compensation)
  std::unique_ptr<b2s_cloud> odo_in;   // de-skewed input of the odometry (allocated when de-skew is first enabled)
  std::unique_ptr<b2s_cloud> map_in;   // de-skewed input of the mapper
  b2s::DevBuf motion;                  // b2s_motion_compensation_result [256], written by the de-skew kernels
  b2s::DevBuf res;                    // b2s_result [2]: the odometry registration, the mapper registration of the step in flight
  b2s::DevBuf odo_slots, slam_slots;   // 256 result slots of each kind
  b2s::DevBuf lookup;                  // b2s_odometry_lookup: 4x4 + has
  b2s::PinnedBuf inputs;               // OdoStepInput ring, device-mapped
  long long host_step = 0;
  bool has_t = false;
  long long last_t = 0;
  bool graph_mode = false;
  struct SlamGraph {
    b2s::GraphCache g;
    double min_fitness = 0.0;
    int ignore_fitness = 0;
  };
  std::map<unsigned long long, SlamGraph> graphs;   // per submap uid; entries of destroyed submaps go when a new submap is added
};

namespace b2s {

__device__ void mat_identity(double* M) {
  for (int i = 0; i < 16; i++) M[i] = (i % 5 == 0) ? 1.0 : 0.0;
}
// Eigen: product of two isometries (linear * linear, linear * translation + translation), row-major 4x4
__device__ void iso_mul(const double* A, const double* B, double* C) {
  double R[16];
  for (int i = 0; i < 3; i++) {
    for (int j = 0; j < 3; j++) R[4 * i + j] = A[4 * i] * B[j] + A[4 * i + 1] * B[4 + j] + A[4 * i + 2] * B[8 + j];
    R[4 * i + 3] = (A[4 * i] * B[3] + A[4 * i + 1] * B[7] + A[4 * i + 2] * B[11]) + A[4 * i + 3];
  }
  R[12] = R[13] = R[14] = 0.0; R[15] = 1.0;
  for (int i = 0; i < 16; i++) C[i] = R[i];
}
// Eigen: inverse of an isometry = (R^T, -(R^T t))
__device__ void iso_inv(const double* A, double* B) {
  double R[16];
  for (int i = 0; i < 3; i++) {
    for (int j = 0; j < 3; j++) R[4 * i + j] = A[4 * j + i];
    R[4 * i + 3] = -(A[i] * A[3] + A[4 + i] * A[7] + A[8 + i] * A[11]);
  }
  R[12] = R[13] = R[14] = 0.0; R[15] = 1.0;
  for (int i = 0; i < 16; i++) B[i] = R[i];
}

// Eigen's Quaterniond(const Matrix3d&) (quaternionbase_assign_impl), q = (x, y, z, w)
__device__ void quat_from_rot(const double* T, double* q) {
  auto m = [T](int i, int j) { return T[4 * i + j]; };
  double t = m(0, 0) + m(1, 1) + m(2, 2);
  if (t > 0.0) {
    t = sqrt(t + 1.0);
    q[3] = 0.5 * t;
    t = 0.5 / t;
    q[0] = (m(2, 1) - m(1, 2)) * t;
    q[1] = (m(0, 2) - m(2, 0)) * t;
    q[2] = (m(1, 0) - m(0, 1)) * t;
  } else {
    int i = 0;
    if (m(1, 1) > m(0, 0)) i = 1;
    if (m(2, 2) > m(i, i)) i = 2;
    const int j = (i + 1) % 3, k = (j + 1) % 3;
    t = sqrt(m(i, i) - m(j, j) - m(k, k) + 1.0);
    q[i] = 0.5 * t;
    t = 0.5 / t;
    q[3] = (m(k, j) - m(j, k)) * t;
    q[j] = (m(j, i) + m(i, j)) * t;
    q[k] = (m(k, i) + m(i, k)) * t;
  }
}
// Eigen's QuaternionBase::toRotationMatrix into the rotation block of T
__device__ void rot_from_quat(const double* q, double* T) {
  const double tx = 2.0 * q[0], ty = 2.0 * q[1], tz = 2.0 * q[2];
  const double twx = tx * q[3], twy = ty * q[3], twz = tz * q[3];
  const double txx = tx * q[0], txy = ty * q[0], txz = tz * q[0];
  const double tyy = ty * q[1], tyz = tz * q[1], tzz = tz * q[2];
  T[0] = 1.0 - (tyy + tzz); T[1] = txy - twz; T[2] = txz + twy;
  T[4] = txy + twz; T[5] = 1.0 - (txx + tzz); T[6] = tyz - twx;
  T[8] = txz - twy; T[9] = tyz + twx; T[10] = 1.0 - (txx + tyy);
}

// interpolate(start, end, time) of Transform.cpp:16-41: translation linear, rotation Eigen slerp, factor over (duration + 1e-6 s)
__device__ void interpolate_dev(const double* A, long long ta, const double* B, long long tb, long long t, double* out) {
  const double duration = (double)(tb - ta) / 1e7;   // toSeconds: ticks of 100 ns
  const double factor = ((double)(t - ta) / 1e7) / (duration + 1e-6);
  double qa[4], qb[4];
  quat_from_rot(A, qa);
  quat_from_rot(B, qb);
  const double one = 1.0 - 2.220446049250313e-16;   // 1 - NumTraits<double>::epsilon()
  const double d = qa[0] * qb[0] + qa[1] * qb[1] + qa[2] * qb[2] + qa[3] * qb[3];
  const double absD = fabs(d);
  double s0, s1;
  if (absD >= one) {
    s0 = 1.0 - factor;
    s1 = factor;
  } else {
    const double theta = acos(absD);
    const double sinTheta = sin(theta);
    s0 = sin((1.0 - factor) * theta) / sinTheta;
    s1 = sin(factor * theta) / sinTheta;
  }
  if (d < 0.0) s1 = -s1;
  double q[4];
  for (int i = 0; i < 4; i++) q[i] = s0 * qa[i] + s1 * qb[i];
  mat_identity(out);
  rot_from_quat(q, out);
  for (int i = 0; i < 3; i++) out[4 * i + 3] = A[4 * i + 3] + (B[4 * i + 3] - A[4 * i + 3]) * factor;
}

struct BufferView {
  const long long* t;
  const double* T;
  int cap, head, count;
  __device__ int phys(int i) const { return (head + i) % cap; }
  __device__ long long time(int i) const { return t[phys(i)]; }
  __device__ const double* tf(int i) const { return T + 16 * phys(i); }
  __device__ bool has(long long q) const { return count > 0 && time(0) <= q && q <= time(count - 1); }
  // getTransform(q, buffer) (TransformInterpolationBuffer.cpp:149-157 -> lookup :83-109); Identity for an empty buffer.  The times
  // never decrease (the mapper's buffer accepts an equal time): the first entry with q <= time is the one std::find_if returns
  __device__ void get(long long q, double* out) const {
    if (count == 0) { mat_identity(out); return; }
    int i = 0;
    if (count > 1) {
      if (q < time(0)) q = time(0);
      if (q > time(count - 1)) q = time(count - 1);
      int lo = 0, hi = count - 1;
      while (lo < hi) { const int mid = (lo + hi) / 2; if (q <= time(mid)) hi = mid; else lo = mid + 1; }
      if (time(lo) != q) { interpolate_dev(tf(lo - 1), time(lo - 1), tf(lo), time(lo), q, out); return; }
      i = lo;
    }
    for (int k = 0; k < 16; k++) out[k] = tf(i)[k];
  }
  // push (TransformInterpolationBuffer.cpp:21-43, 111-115): a time earlier than the earliest or the latest entry is ignored, then
  // push_back and pop_front while the size exceeds the limit.  Updates head / count of the caller's state.
  __device__ static void push(long long* rt, double* rT, int cap, int32_t* head, int32_t* count, long long t, const double* T) {
    if (*count > 0 && (t < rt[*head] || t < rt[(*head + *count - 1) % cap])) return;
    int idx;
    if (*count < cap) { idx = (*head + *count) % cap; *count += 1; }
    else { idx = *head; *head = (*head + 1) % cap; }
    rt[idx] = t;
    for (int i = 0; i < 16; i++) rT[16 * idx + i] = T[i];
  }
  // ConstantVelocityMotionCompensation::estimateLinearAndAngularVelocity (MotionCompensation.cpp:32-57) at time q
  __device__ void velocity(long long q, int offset, double* v, double* w) const {
    for (int k = 0; k < 3; k++) v[k] = w[k] = 0.0;
    if (count <= offset || !(time(count - 1) < q)) return;   // too few poses / "buffer has this already": zeros
    const int fi = count - 1, si = count - 1 - offset;
    double Si[16], dT[16];
    iso_inv(tf(si), Si);
    iso_mul(Si, tf(fi), dT);
    const double dt = (double)(time(fi) - time(si)) / 1e7;
    double qq[4];
    quat_from_rot(dT, qq);
    for (int pass = 0; pass < 2; pass++) {   // Quaterniond(...).normalized(), then toRPY's own normalize() (math.cpp:39-41)
      const double z = qq[0] * qq[0] + qq[1] * qq[1] + qq[2] * qq[2] + qq[3] * qq[3];
      if (z > 0.0) { const double n = sqrt(z); for (int k = 0; k < 4; k++) qq[k] /= n; }
    }
    const double x = qq[0], y = qq[1], z = qq[2], ww = qq[3];
    const double den = dt + 1e-6;
    for (int k = 0; k < 3; k++) v[k] = dT[4 * k + 3] / den;
    w[0] = atan2(2 * (ww * x + y * z), 1 - 2 * (x * x + y * y)) / den;   // getRollFromQuat (math.hpp:30-42)
    w[1] = asin(2 * (ww * y - x * z)) / den;
    w[2] = atan2(2 * (ww * z + x * y), 1 - 2 * (y * y + z * z)) / den;
  }
};

__device__ BufferView buffer_view(const OdoState* s, const long long* rt, const double* rT, int cap) {
  BufferView b;
  b.t = rt; b.T = rT; b.cap = cap; b.head = s->head; b.count = s->count;
  return b;
}
// the mapper's mapToRangeSensorBuffer_
__device__ BufferView map_view(const OdoState* s, const long long* rt, const double* rT, int cap) {
  BufferView b;
  b.t = rt; b.T = rT; b.cap = cap; b.head = s->map_head; b.count = s->map_count;
  return b;
}

constexpr int DESKEW_THREADS = 256;

// D2: one de-skew of the step in flight.  Thread 0 of every CTA estimates the velocities from the buffer (odometry's or mapper's) at
// the step's timestamp and shares them; every thread then moves its points with undistort_point.  CTA 0 records the velocities in the
// step's result slot.  The count is read on the device, the launch is sized by the caller's bound, so the launch can be captured.
__global__ void __launch_bounds__(DESKEW_THREADS) deskew_kernel(const double* __restrict__ xyz, const int32_t* __restrict__ d_n, const OdoState* s,
                                                                const long long* __restrict__ rt, const double* __restrict__ rT, int cap, int map,
                                                                double duration, int clockwise, int offset, double* __restrict__ out, int32_t* out_n,
                                                                b2s_motion_compensation_result* rec) {
  pdl_wait();
  __shared__ double vel[6];
  if (threadIdx.x == 0) {
    const BufferView b = map ? map_view(s, rt, rT, cap) : buffer_view(s, rt, rT, cap);
    b.velocity(s->t_cur, offset, vel, vel + 3);
    if (blockIdx.x == 0) {
      b2s_motion_compensation_result* o = rec + s->slot;
      double* v = map ? o->map_linear_velocity : o->odometry_linear_velocity;
      double* w = map ? o->map_angular_velocity_rpy : o->odometry_angular_velocity_rpy;
      int applied = 0;
      for (int k = 0; k < 3; k++) {
        v[k] = vel[k]; w[k] = vel[3 + k];
        applied |= vel[k] != 0.0 || vel[3 + k] != 0.0;
      }
      if (map) o->map_applied = applied; else o->odometry_applied = applied;
      *out_n = *d_n;
    }
  }
  __syncthreads();
  const int n = *d_n;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x)
    undistort_point(xyz[3 * i], xyz[3 * i + 1], xyz[3 * i + 2], vel[0], vel[1], vel[2], vel[3], vel[4], vel[5], duration, clockwise, out + 3 * i);
}

__global__ void map_pose_push_kernel(OdoState* s, long long* map_t, double* map_T, int cap, long long t, Mat16 T) {
  pdl_wait();
  if (threadIdx.x != 0) return;
  BufferView::push(map_t, map_T, cap, &s->map_head, &s->map_count, t, T.v);
}

// first node of every odometry step: this step's timestamp and result slot from the host ring
__global__ void odometry_begin_kernel(const OdoStepInput* __restrict__ inputs, OdoState* s) {
  pdl_wait();
  if (threadIdx.x != 0) return;
  const int step = s->step;
  const OdoStepInput in = inputs[step & (ODO_RING - 1)];
  s->t_cur = in.t;
  s->slot = in.slot;
  s->step = step + 1;
}

// Odometry.cpp:33-79 after the registration: initialise / ok / failed, the cumulative pose, the buffer push, the result slot
__global__ void odometry_gate_kernel(const b2s_result* __restrict__ reg, const int32_t* __restrict__ prev_n, const int32_t* __restrict__ pre_n,
                                     double min_fitness, int cap, OdoState* s, long long* ring_t, double* ring_T, b2s_odometry_result* slots) {
  pdl_wait();
  if (threadIdx.x != 0) return;
  const int np = *prev_n, nq = *pre_n;
  int outcome;
  bool push = false;
  if (np == 0) {                                  // cloudPrev_.IsEmpty(): cloudPrev_ = pre, push
    outcome = B2S_ODOM_INIT;
    push = true;
    s->keep = 1;
  } else if (reg->fitness > min_fitness) {        // isOdomOkay
    if (s->init_pending) {
      for (int i = 0; i < 16; i++) s->cum[i] = s->init_T[i];
      s->init_pending = 0;
    } else {
      double inv[16];
      iso_inv(reg->T, inv);
      iso_mul(s->cum, inv, s->cum);
    }
    outcome = B2S_ODOM_OK;
    push = true;
    s->keep = 1;
  } else {                                        // failed: keep the previous cloud only when the new one is empty
    outcome = nq > 0 ? B2S_ODOM_FAILED : B2S_ODOM_FAILED_KEPT_PREV;
    s->keep = nq > 0;
  }
  if (push) {   // push_back, then pop_front while the size exceeds the limit
    int idx;
    if (s->count < cap) { idx = (s->head + s->count) % cap; s->count += 1; }
    else { idx = s->head; s->head = (s->head + 1) % cap; }
    ring_t[idx] = s->t_cur;
    for (int i = 0; i < 16; i++) ring_T[16 * idx + i] = s->cum[i];
  }
  b2s_odometry_result* o = slots + s->slot;
  if (outcome == B2S_ODOM_INIT) memset(&o->registration, 0, sizeof(b2s_result));
  else o->registration = *reg;
  for (int i = 0; i < 16; i++) o->odom_to_range_sensor[i] = s->cum[i];
  o->outcome = outcome;
  o->n_preprocessed = nq;
}

// cloudPrev_ = pre when the gate said so: a copy of the device-side count, so the captured launch never changes
__global__ void odometry_keep_kernel(const double* __restrict__ pre_xyz, const double* __restrict__ pre_nrm, const int32_t* __restrict__ pre_n,
                                     double* __restrict__ prev_xyz, double* __restrict__ prev_nrm, int32_t* prev_n, const OdoState* __restrict__ s) {
  pdl_wait();
  if (!s->keep) return;
  const int n = *pre_n;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < 3 * n; i += gridDim.x * blockDim.x) {
    prev_xyz[i] = pre_xyz[i];
    prev_nrm[i] = pre_nrm[i];
  }
  if (blockIdx.x == 0 && threadIdx.x == 0) *prev_n = n;
}

// Mapper.cpp:122-137: odom_used = has(t); motion = getTransform(t_last)^-1 * getTransform(t); guess = pose * motion
// (pose slots of the submap: [0] mapToRangeSensor_, [2] odometry motion, [3] guess)
// After a new initial value, and in the step after it, the guess is the pose itself (Mapper.cpp:130-138; ms: the submap's MS_* words)
__global__ void odometry_prediction_kernel(OdoState* s, const long long* __restrict__ ring_t, const double* __restrict__ ring_T, int cap, double* pose,
                                           const int32_t* __restrict__ ms) {
  pdl_wait();
  if (threadIdx.x != 0) return;
  const bool hold = ms[MS_NEWINIT] || ms[MS_IGNODOM];
  const BufferView b = buffer_view(s, ring_t, ring_T, cap);
  const bool used = b.has(s->t_cur);
  double M[16];
  mat_identity(M);
  if (used) {
    double A[16], B[16], Ai[16];
    b.get(s->t_last, A);
    b.get(s->t_cur, B);
    iso_inv(A, Ai);
    iso_mul(Ai, B, M);
  }
  for (int i = 0; i < 16; i++) pose[32 + i] = M[i];
  double G[16];
  for (int i = 0; i < 4; i++)   // the full 4x4 product, as compose_kernel of the host-fed chain computes the guess
    for (int j = 0; j < 4; j++) {
      double acc = 0.0;
      for (int k = 0; k < 4; k++) acc += pose[4 * i + k] * M[4 * k + j];
      G[4 * i + j] = hold ? pose[4 * i + j] : acc;
    }
  for (int i = 0; i < 16; i++) pose[48 + i] = G[i];
  s->odom_used = used;
}

// after the mapper's gate: for an accepted scan mapToRangeSensorBuffer_.push(t, mapToRangeSensor_) (Mapper.cpp:160, pose[0..15] is
// the registration result by now) and lastMeasurementTimestamp_ = t (:164,178); then the combined result slot.  The first step after a
// new initial value pushes the pose it kept and leaves lastMeasurementTimestamp_ alone (:143-149)
__global__ void slam_post_kernel(OdoState* s, const int32_t* __restrict__ ms, const b2s_result* __restrict__ mres,
                                 const b2s_odometry_result* __restrict__ odo_slots, b2s_slam_result* slam_slots, const double* __restrict__ pose,
                                 long long* map_t, double* map_T, int cap) {
  pdl_wait();
  if (threadIdx.x != 0) return;
  const int accepted = ms[MS_ACCEPT];
  if (accepted) {
    BufferView::push(map_t, map_T, cap, &s->map_head, &s->map_count, s->t_cur, pose);
    if (!ms[MS_INITSTEP]) s->t_last = s->t_cur;
  }
  b2s_slam_result* o = slam_slots + s->slot;
  o->odometry = odo_slots[s->slot];
  o->mapper = *mres;
  o->odom_used = s->odom_used;
  o->mapper_accepted = accepted;
}

__global__ void odometry_set_initial_kernel(OdoState* s, Mat16 T) {
  pdl_wait();
  if (threadIdx.x < 16) { s->cum[threadIdx.x] = T.v[threadIdx.x]; s->init_T[threadIdx.x] = T.v[threadIdx.x]; }
  if (threadIdx.x == 0) s->init_pending = 1;
}

__global__ void odometry_lookup_kernel(const OdoState* s, const long long* __restrict__ ring_t, const double* __restrict__ ring_T, int cap, long long t,
                                       double* out, int map) {
  pdl_wait();
  if (threadIdx.x != 0) return;
  const BufferView b = map ? map_view(s, ring_t, ring_T, cap) : buffer_view(s, ring_t, ring_T, cap);
  b.get(t, out);
  out[16] = b.has(t) ? 1.0 : 0.0;
}

static int32_t check_odometry_params(const b2s_odometry_params& p) {
  B2S_TRY(check_icp_params(p.icp));
  B2S_REQUIRE(p.downsampling_ratio >= 0.0 && p.downsampling_ratio <= 1.0, B2S_E_INVALID, "[RandomDownSample] sampling_ratio must be in [0, 1]");
  B2S_REQUIRE(p.voxel_size >= 0.0, B2S_E_INVALID, "voxel size must be >= 0");
  B2S_REQUIRE(p.buffer_size >= 1, B2S_E_INVALID, "buffer_size must be >= 1");
  B2S_REQUIRE(p.min_fitness == p.min_fitness, B2S_E_INVALID, "min_fitness is NaN");
  return B2S_OK;
}

// checks shared by every step: the timestamp order, then the step's entry of the host ring (read by odometry_begin_kernel)
static int32_t odometry_push_input(b2s_handle* h, b2s_odometry* od, long long t, int32_t slot) {
  B2S_REQUIRE(!od->has_t || t > od->last_t, B2S_E_INVALID, "odometry: timestamp %lld is not after the previous one (%lld)", t, od->last_t);
  // the ring has 64 entries and the host may run ahead of the device: never by more than 32 steps
  if ((od->host_step & 31) == 0) B2S_CUDA(cudaStreamSynchronize(h->stream));
  OdoStepInput* in = od->inputs.as<OdoStepInput>() + (od->host_step & (ODO_RING - 1));
  in->t = t; in->slot = slot; in->pad = 0;
  od->host_step++;
  od->has_t = true;
  od->last_t = t;
  return B2S_OK;
}

// D2: raw -> out de-skewed with the velocities of the odometry's buffer (map = false) or the mapper's (map = true), one launch sized by
// raw's bound (the staging capacity in graph mode)
static int32_t deskew(b2s_handle* h, b2s_odometry* od, const b2s_cloud* raw, bool map, b2s_cloud* out) {
  const b2s_motion_compensation_params& mc = od->mc;
  out->fixed_cap = raw->fixed_cap;   // downstream sizing sees what it would see on raw: a staging cloud's bound, never its last count
  out->n_max = raw->n_max;
  out->n_known = raw->n_known;
  out->has_normals = false;   // the reference copies the input cloud and rewrites points_ only
  launch_pdl(deskew_kernel, grid_for(raw->n_max, DESKEW_THREADS), DESKEW_THREADS, 0, h->stream, raw->xyz.as<double>(), raw->dn.as<int32_t>(),
             od->state.as<OdoState>(), (map ? od->map_t : od->ring_t).as<long long>(), (map ? od->map_T : od->ring_T).as<double>(),
             od->params.buffer_size, map ? 1 : 0, mc.scan_duration, mc.spinning_clockwise ? 1 : 0, mc.num_poses_velocity_estimation,
             out->xyz.as<double>(), out->dn.as<int32_t>(), od->motion.as<b2s_motion_compensation_result>());
  h->launches++;
  return B2S_OK;
}

// Odometry.cpp:25-79 on the device, reading the step's inputs from the host ring; with de-skew enabled the odometry works on the scan
// de-skewed from its own buffer (SlamWrapper.cpp:266-268)
static int32_t odometry_chain(b2s_handle* h, b2s_odometry* od, const b2s_cloud* raw) {
  const b2s_odometry_params& p = od->params;
  OdoState* s = od->state.as<OdoState>();
  OdoStepInput* inputs_dev = nullptr;
  B2S_CUDA(cudaHostGetDevicePointer(reinterpret_cast<void**>(&inputs_dev), od->inputs.p, 0));
  launch_pdl(odometry_begin_kernel, 1, 32, 0, h->stream, inputs_dev, s);
  h->launches++;
  if (od->mc.enabled) {
    B2S_TRY(deskew(h, od, raw, false, od->odo_in.get()));
    raw = od->odo_in.get();
  }
  b2s_cloud* pre = od->pre.get();
  b2s_cloud* prev = od->prev.get();
  B2S_TRY(preprocess_scan(h, raw, p.cropper, p.voxel_size, p.downsampling_ratio, p.seed, p.icp, od->scratch.get(), pre));   // :25-30
  // registerClouds(cloudPrev_, pre, Identity) (:48): source = the previous cloud, target = the current one, indexed every step
  B2S_TRY(grid_build(h, &od->grid, pre, nn_cell(h, p.icp.max_corr_dist), nullptr));
  B2S_TRY(h->work_xyz.ensure(icp_work_bytes(prev->n_max), h->stream));
  b2s_result* reg = od->res.as<b2s_result>();
  const double I[16] = {1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1};
  IcpProblem P;
  fill_problem(&P, p.icp, prev, &od->grid, pre, I, nullptr, h->work_xyz.as<double>(), reg);
  B2S_TRY(icp_launch(h, &P, nullptr, 1, prev->n_max));
  launch_pdl(odometry_gate_kernel, 1, 32, 0, h->stream, reg, prev->dn.as<int32_t>(), pre->dn.as<int32_t>(), p.min_fitness, p.buffer_size, s,
             od->ring_t.as<long long>(), od->ring_T.as<double>(), od->odo_slots.as<b2s_odometry_result>());
  launch_pdl(odometry_keep_kernel, grid_for(3 * od->capacity, 256), 256, 0, h->stream, pre->xyz.as<double>(), pre->nrm.as<double>(),
             pre->dn.as<int32_t>(), prev->xyz.as<double>(), prev->nrm.as<double>(), prev->dn.as<int32_t>(), s);
  h->launches += 2;
  prev->n_known = -1;
  B2S_CUDA(cudaGetLastError());
  return B2S_OK;
}

struct SlamCtx {
  b2s_handle* h; b2s_submap* sm; b2s_odometry* od; const b2s_cloud* raw; double min_fitness; int ignore_fitness;
};

// odometry, the prediction from its buffer, then the mapper chain (S1 -> S2 -> gates -> [carving] -> F1 -> [dense map]), the mapper's
// pose buffer and t_last.  With de-skew enabled the mapper chain works on the scan de-skewed from the mapper's buffer
// (SlamWrapper.cpp:298-304): it is the raw scan of pre-processing, ICP, carving and the dense map
static int32_t slam_chain(void* ctx) {
  const SlamCtx& c = *static_cast<const SlamCtx*>(ctx);
  b2s_handle* h = c.h;
  b2s_odometry* od = c.od;
  b2s_submap* sm = c.sm;
  B2S_TRY(odometry_chain(h, od, c.raw));
  OdoState* s = od->state.as<OdoState>();
  double* pose_state = sm->pose.as<double>();
  b2s_result* mres = od->res.as<b2s_result>() + 1;
  const b2s_cloud* raw = c.raw;
  if (od->mc.enabled) {
    B2S_TRY(deskew(h, od, raw, true, od->map_in.get()));
    raw = od->map_in.get();
  }
  launch_pdl(odometry_prediction_kernel, 1, 32, 0, h->stream, s, od->ring_t.as<long long>(), od->ring_T.as<double>(), od->params.buffer_size,
             pose_state, static_cast<const int32_t*>(sm->mstate.as<int32_t>()));
  h->launches++;
  B2S_TRY(process_scan_impl(h, raw, h->t1.get(), h->t2.get()));                                                   // Mapper.cpp:139
  B2S_TRY(register_to_submap_async(h, h->t2.get(), sm, nullptr, pose_state, nullptr, pose_state + 48, mres));   // Mapper.cpp:140-141
  B2S_TRY(mapper_chain_tail(h, sm, raw, h->t1.get(), mres, c.min_fitness, c.ignore_fitness, nullptr, nullptr));   // Mapper.cpp:151-177
  launch_pdl(slam_post_kernel, 1, 32, 0, h->stream, s, sm->mstate.as<int32_t>(), mres, od->odo_slots.as<b2s_odometry_result>(),
             od->slam_slots.as<b2s_slam_result>(), static_cast<const double*>(pose_state), od->map_t.as<long long>(), od->map_T.as<double>(),
             od->params.buffer_size);
  h->launches++;
  B2S_CUDA(cudaGetLastError());
  return B2S_OK;
}

static int32_t check_raw(const b2s_odometry* od, const b2s_cloud* raw) {
  B2S_REQUIRE(raw->h == od->h, B2S_E_INVALID, "the scan belongs to another handle");
  B2S_REQUIRE(raw->n_max <= od->capacity, B2S_E_CAPACITY, "scan of up to %zu points, the odometry holds %zu", raw->n_max, od->capacity);
  return B2S_OK;
}

// getTransform(t) / has(t) of the odometry's buffer or the mapper's; the caller holds the lock
static int32_t buffer_lookup(b2s_handle* h, const b2s_odometry* od, bool map, long long t, double T[16], int32_t* has) {
  launch_pdl(odometry_lookup_kernel, 1, 32, 0, h->stream, od->state.as<OdoState>(), (map ? od->map_t : od->ring_t).as<long long>(),
             (map ? od->map_T : od->ring_T).as<double>(), od->params.buffer_size, t, od->lookup.as<double>(), map ? 1 : 0);
  h->launches++;
  B2S_CUDA(cudaGetLastError());
  double v[17];
  B2S_TRY(read_back(h, {{v, od->lookup.p, sizeof(v)}}));
  memcpy(T, v, 128);
  if (has) *has = v[16] != 0.0;
  return B2S_OK;
}

// b2s_odometry_create's set-up of a new object
static int32_t odometry_init(b2s_handle* h, b2s_odometry* od, const b2s_odometry_params* p, size_t capacity_points) {
  od->h = h;
  od->device = h->device;
  od->params = *p;
  od->capacity = capacity_points;
  B2S_TRY(make_cloud(h, capacity_points, true, true, &od->prev));
  od->prev->has_normals = true;
  B2S_TRY(make_cloud(h, 1, true, false, &od->pre));
  B2S_TRY(make_cloud(h, 1, true, false, &od->scratch));
  B2S_TRY(make_cloud(h, 1, false, false, &od->input));
  B2S_TRY(od->state.ensure(sizeof(OdoState), h->stream));
  B2S_CUDA(cudaMemsetAsync(od->state.p, 0, sizeof(OdoState), h->stream));
  const double I[16] = {1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1};
  B2S_TRY(pose_to_device(h, I, od->state.as<OdoState>()->cum));
  B2S_TRY(od->ring_t.ensure((size_t)p->buffer_size * 8, h->stream));
  B2S_TRY(od->ring_T.ensure((size_t)p->buffer_size * 128, h->stream));
  B2S_TRY(od->map_t.ensure((size_t)p->buffer_size * 8, h->stream));
  B2S_TRY(od->map_T.ensure((size_t)p->buffer_size * 128, h->stream));
  b2s_default_motion_compensation_params(&od->mc);
  B2S_TRY(od->res.ensure(2 * sizeof(b2s_result), h->stream));
  B2S_CUDA(cudaMemsetAsync(od->res.p, 0, 2 * sizeof(b2s_result), h->stream));
  B2S_TRY(od->odo_slots.ensure(256 * sizeof(b2s_odometry_result), h->stream));
  B2S_CUDA(cudaMemsetAsync(od->odo_slots.p, 0, 256 * sizeof(b2s_odometry_result), h->stream));
  B2S_TRY(od->slam_slots.ensure(256 * sizeof(b2s_slam_result), h->stream));
  B2S_CUDA(cudaMemsetAsync(od->slam_slots.p, 0, 256 * sizeof(b2s_slam_result), h->stream));
  B2S_TRY(od->lookup.ensure(17 * 8, h->stream));
  B2S_TRY(od->inputs.alloc(ODO_RING * sizeof(OdoStepInput), cudaHostAllocMapped));
  memset(od->inputs.p, 0, ODO_RING * sizeof(OdoStepInput));
  return B2S_OK;
}

// the two de-skewed clouds and the velocity records, allocated when de-skew is first enabled
static int32_t odometry_deskew_buffers(b2s_handle* h, b2s_odometry* od) {
  if (od->odo_in) return B2S_OK;
  std::unique_ptr<b2s_cloud> a, b;
  B2S_TRY(make_cloud(h, od->capacity, false, false, &a));
  B2S_TRY(make_cloud(h, od->capacity, false, false, &b));
  B2S_TRY(od->motion.ensure(256 * sizeof(b2s_motion_compensation_result), h->stream));
  B2S_CUDA(cudaMemsetAsync(od->motion.p, 0, 256 * sizeof(b2s_motion_compensation_result), h->stream));
  od->odo_in = std::move(a);
  od->map_in = std::move(b);
  return B2S_OK;
}

}  // namespace b2s

extern "C" {

void b2s_default_odometry_params(b2s_odometry_params* p) {
  memset(p, 0, sizeof(*p));
  b2s_config cfg;
  b2s_default_config(&cfg);
  p->icp = cfg.icp;
  p->voxel_size = cfg.scan.voxel_size;
  p->downsampling_ratio = cfg.scan.downsampling_ratio;
  p->seed = cfg.scan.seed;
  p->cropper = cfg.scan.scan_matcher_cropper;
  p->min_fitness = 0.1;
  p->buffer_size = 2000;
}

int32_t b2s_odometry_create(b2s_handle* h, const b2s_odometry_params* p, size_t capacity_points, b2s_odometry** out) {
  B2S_REQUIRE(h && p && out && capacity_points > 0, B2S_E_INVALID, "bad argument");
  B2S_REQUIRE(capacity_points < (size_t)0x7fffffff / 4, B2S_E_INVALID, "capacity too large");
  B2S_TRY(check_odometry_params(*p));
  LOCK(h);
  return create_object(out, [&](b2s_odometry* od) -> int32_t { return odometry_init(h, od, p, capacity_points); });
}

void b2s_odometry_destroy(b2s_odometry* od) { destroy_object(od); }

int32_t b2s_odometry_set_params(b2s_handle* h, b2s_odometry* od, const b2s_odometry_params* p) {
  B2S_REQUIRE(h && od && p, B2S_E_INVALID, "null argument");
  B2S_REQUIRE(od->h == h, B2S_E_INVALID, "the odometry belongs to another handle");
  B2S_TRY(check_odometry_params(*p));
  B2S_REQUIRE(p->buffer_size == od->params.buffer_size, B2S_E_INVALID, "buffer_size is fixed at creation (%d)", (int)od->params.buffer_size);
  LOCK(h);
  od->params = *p;
  od->params_gen++;
  return B2S_OK;
}

int32_t b2s_odometry_set_initial_transform(b2s_handle* h, b2s_odometry* od, const double T[16]) {
  B2S_REQUIRE(h && od && T, B2S_E_INVALID, "null argument");
  B2S_REQUIRE(od->h == h, B2S_E_INVALID, "the odometry belongs to another handle");
  LOCK(h);
  Mat16 m;
  memcpy(m.v, T, sizeof(m.v));
  launch_pdl(odometry_set_initial_kernel, 1, 32, 0, h->stream, od->state.as<OdoState>(), m);
  h->launches++;
  B2S_CUDA(cudaGetLastError());
  return B2S_OK;
}

int32_t b2s_odometry_step_async(b2s_handle* h, b2s_odometry* od, const b2s_cloud* raw, int64_t t, int32_t slot) {
  B2S_REQUIRE(h && od && raw, B2S_E_INVALID, "null argument");
  B2S_REQUIRE(od->h == h, B2S_E_INVALID, "the odometry belongs to another handle");
  B2S_REQUIRE(slot >= 0 && slot < 256, B2S_E_INVALID, "slot out of range");
  B2S_TRY(check_raw(od, raw));
  LOCK(h);
  B2S_TRY(odometry_push_input(h, od, t, slot));
  PdlScope pdl;
  return odometry_chain(h, od, raw);
}

int32_t b2s_odometry_result_fetch(b2s_handle* h, b2s_odometry* od, int32_t slot, b2s_odometry_result* out) {
  B2S_REQUIRE(h && od && out && slot >= 0 && slot < 256, B2S_E_INVALID, "bad argument");
  B2S_REQUIRE(od->h == h, B2S_E_INVALID, "the odometry belongs to another handle");
  LOCK(h);
  return read_back(h, {{out, od->odo_slots.as<b2s_odometry_result>() + slot, sizeof(b2s_odometry_result)}});
}

int32_t b2s_odometry_lookup(b2s_handle* h, const b2s_odometry* od, int64_t t, double T[16], int32_t* has) {
  B2S_REQUIRE(h && od && T, B2S_E_INVALID, "null argument");
  B2S_REQUIRE(od->h == h, B2S_E_INVALID, "the odometry belongs to another handle");
  LOCK(h);
  return buffer_lookup(h, od, false, t, T, has);
}

int32_t b2s_odometry_preprocessed(b2s_handle* h, const b2s_odometry* od, b2s_cloud* out) {
  B2S_REQUIRE(h && od && out, B2S_E_INVALID, "null argument");
  B2S_REQUIRE(od->h == h && out->h == h, B2S_E_INVALID, "the odometry or the cloud belongs to another handle");
  LOCK(h);
  return op_voxel_down_sample(h, od->prev.get(), nullptr, 0.0, out);   // voxel <= 0: plain device copy
}

static int32_t slam_step(b2s_handle* h, b2s_submap* sm, b2s_odometry* od, const b2s_cloud* raw, long long t, double min_fitness, int32_t ignore,
                         int32_t slot) {
  B2S_REQUIRE(sm->h == h && od->h == h, B2S_E_INVALID, "the submap or the odometry belongs to another handle");
  B2S_REQUIRE(slot >= 0 && slot < 256, B2S_E_INVALID, "slot out of range");
  B2S_REQUIRE(!od->graph_mode || raw == od->staging.get(), B2S_E_INVALID,
              "graph mode: the scan must be uploaded into the staging cloud of b2s_slam_graph_enable");
  B2S_TRY(check_raw(od, raw));
  B2S_TRY(odometry_push_input(h, od, t, slot));
  PdlScope pdl;   // the chain's launches (eager and captured) overlap their predecessors' tails: see pdl_wait in common.cuh
  SlamCtx ctx{h, sm, od, raw, min_fitness, ignore};
  if (!od->graph_mode) return slam_chain(&ctx);
  sm->fixed_launch = true;   // the submap's fusion and carving size their launches for a captured chain from now on
  if (od->graphs.find(sm->uid) == od->graphs.end()) {   // a submap seen for the first time: forget the graphs of destroyed submaps
    for (auto it = od->graphs.begin(); it != od->graphs.end();) it = submap_alive(it->first) ? std::next(it) : od->graphs.erase(it);
  }
  b2s_odometry::SlamGraph& g = od->graphs[sm->uid];
  if (g.min_fitness != min_fitness || g.ignore_fitness != ignore) {
    B2S_TRY(graph_drop(h, &g.g));
    g.min_fitness = min_fitness;
    g.ignore_fitness = ignore;
  }
  // the options of this submap and the odometry's parameters are baked into the captured launches
  return graph_step(h, &g.g, (od->params_gen << 32) ^ sm->opts_gen, slam_chain, &ctx);
}

int32_t b2s_slam_step_async(b2s_handle* h, b2s_submap* sm, b2s_odometry* od, const b2s_cloud* raw, int64_t t, double min_refinement_fitness,
                            int32_t ignore_min_fitness, int32_t slot) {
  B2S_REQUIRE(h && sm && od && raw, B2S_E_INVALID, "null argument");
  LOCK(h);
  return slam_step(h, sm, od, raw, t, min_refinement_fitness, ignore_min_fitness, slot);
}

int32_t b2s_slam_result_fetch(b2s_handle* h, b2s_odometry* od, int32_t slot, b2s_slam_result* out) {
  B2S_REQUIRE(h && od && out && slot >= 0 && slot < 256, B2S_E_INVALID, "bad argument");
  B2S_REQUIRE(od->h == h, B2S_E_INVALID, "the odometry belongs to another handle");
  LOCK(h);
  return read_back(h, {{out, od->slam_slots.as<b2s_slam_result>() + slot, sizeof(b2s_slam_result)}});
}

int32_t b2s_slam_step_host_async(b2s_handle* h, b2s_submap* sm, b2s_odometry* od, const void* xyz_f32, size_t n, size_t stride_bytes, int64_t t,
                                 double min_refinement_fitness, int32_t ignore_min_fitness, b2s_slam_result* out_pinned) {
  B2S_REQUIRE(h && sm && od && xyz_f32 && out_pinned, B2S_E_INVALID, "null argument");
  B2S_REQUIRE(od->h == h, B2S_E_INVALID, "the odometry belongs to another handle");
  B2S_REQUIRE(n <= od->capacity, B2S_E_CAPACITY, "scan of %zu points, the odometry holds %zu", n, od->capacity);
  LOCK(h);   // upload + chain + result copy as one unit
  b2s_cloud* dst = od->graph_mode ? od->staging.get() : od->input.get();
  B2S_REQUIRE(!dst->fixed_cap || n <= dst->fixed_cap, B2S_E_CAPACITY, "scan of %zu points, the staging cloud holds %zu", n, dst->fixed_cap);
  B2S_TRY(b2s_cloud_upload_f32(h, dst, xyz_f32, n, stride_bytes));
  const int32_t slot = (int32_t)(od->host_step & 255);
  B2S_TRY(slam_step(h, sm, od, dst, t, min_refinement_fitness, ignore_min_fitness, slot));
  B2S_CUDA(cudaMemcpyAsync(out_pinned, od->slam_slots.as<b2s_slam_result>() + slot, sizeof(b2s_slam_result), cudaMemcpyDeviceToHost, h->stream));
  return B2S_OK;
}

int32_t b2s_slam_graph_enable(b2s_handle* h, b2s_odometry* od, size_t raw_capacity_points, b2s_cloud** staging_out) {
  B2S_REQUIRE(h && od && staging_out && raw_capacity_points > 0, B2S_E_INVALID, "bad argument");
  B2S_REQUIRE(od->h == h, B2S_E_INVALID, "the odometry belongs to another handle");
  B2S_REQUIRE(raw_capacity_points <= od->capacity, B2S_E_CAPACITY, "staging capacity %zu above the odometry's %zu", raw_capacity_points,
              od->capacity);
  LOCK(h);
  if (!od->staging) B2S_TRY(make_cloud(h, raw_capacity_points, false, true, &od->staging));
  B2S_REQUIRE(od->staging->fixed_cap == raw_capacity_points, B2S_E_INVALID, "the staging cloud already exists with capacity %zu",
              od->staging->fixed_cap);
  od->graph_mode = true;
  *staging_out = od->staging.get();
  return B2S_OK;
}

void b2s_default_motion_compensation_params(b2s_motion_compensation_params* p) {
  memset(p, 0, sizeof(*p));
  p->enabled = 0;
  p->spinning_clockwise = 1;
  p->scan_duration = 0.1;
  p->num_poses_velocity_estimation = 3;
}

int32_t b2s_odometry_set_motion_compensation(b2s_handle* h, b2s_odometry* od, const b2s_motion_compensation_params* p) {
  B2S_REQUIRE(h && od && p, B2S_E_INVALID, "null argument");
  B2S_REQUIRE(od->h == h, B2S_E_INVALID, "the odometry belongs to another handle");
  B2S_REQUIRE(p->scan_duration > 0.0, B2S_E_INVALID, "lidar scanDuration_: must be > 0");   // assert_gt at MotionCompensation.cpp:61
  B2S_REQUIRE(p->num_poses_velocity_estimation >= 1, B2S_E_INVALID, "num_poses_velocity_estimation must be >= 1");
  LOCK(h);
  if (p->enabled) B2S_TRY(odometry_deskew_buffers(h, od));
  od->mc = *p;
  od->params_gen++;   // the captured combined graphs bake the parameters in
  return B2S_OK;
}

int32_t b2s_slam_map_pose_push(b2s_handle* h, b2s_odometry* od, int64_t t, const double T[16]) {
  B2S_REQUIRE(h && od && T, B2S_E_INVALID, "null argument");
  B2S_REQUIRE(od->h == h, B2S_E_INVALID, "the odometry belongs to another handle");
  LOCK(h);
  Mat16 m;
  memcpy(m.v, T, sizeof(m.v));
  launch_pdl(map_pose_push_kernel, 1, 32, 0, h->stream, od->state.as<OdoState>(), od->map_t.as<long long>(), od->map_T.as<double>(),
             od->params.buffer_size, (long long)t, m);
  h->launches++;
  B2S_CUDA(cudaGetLastError());
  return B2S_OK;
}

int32_t b2s_slam_map_lookup(b2s_handle* h, const b2s_odometry* od, int64_t t, double T[16], int32_t* has) {
  B2S_REQUIRE(h && od && T, B2S_E_INVALID, "null argument");
  B2S_REQUIRE(od->h == h, B2S_E_INVALID, "the odometry belongs to another handle");
  LOCK(h);
  return buffer_lookup(h, od, true, t, T, has);
}

int32_t b2s_slam_motion_fetch(b2s_handle* h, b2s_odometry* od, int32_t slot, b2s_motion_compensation_result* out) {
  B2S_REQUIRE(h && od && out && slot >= 0 && slot < 256, B2S_E_INVALID, "bad argument");
  B2S_REQUIRE(od->h == h, B2S_E_INVALID, "the odometry belongs to another handle");
  LOCK(h);   // b2s_odometry_set_motion_compensation allocates the records under the lock
  B2S_REQUIRE(od->motion.p, B2S_E_INVALID, "motion compensation was never enabled on this odometry");
  return read_back(h, {{out, od->motion.as<b2s_motion_compensation_result>() + slot, sizeof(b2s_motion_compensation_result)}});
}

int32_t b2s_slam_undistorted(b2s_handle* h, const b2s_odometry* od, b2s_cloud* odo_out, b2s_cloud* map_out) {
  B2S_REQUIRE(h && od, B2S_E_INVALID, "null argument");
  B2S_REQUIRE(od->h == h && (!odo_out || odo_out->h == h) && (!map_out || map_out->h == h), B2S_E_INVALID,
              "the odometry or a cloud belongs to another handle");
  LOCK(h);
  B2S_REQUIRE(od->odo_in, B2S_E_INVALID, "motion compensation was never enabled on this odometry");
  const b2s_cloud* src[2] = {od->odo_in.get(), od->map_in.get()};
  b2s_cloud* dst[2] = {odo_out, map_out};
  for (int i = 0; i < 2; i++) {
    if (!dst[i]) continue;
    B2S_TRY(op_voxel_down_sample(h, src[i], nullptr, 0.0, dst[i]));   // voxel <= 0: plain device copy
    dst[i]->n_known = -1;   // a replayed graph updates only the device count: the host-side one may be that of the captured step
  }
  return B2S_OK;
}

}  // extern "C"

// ---- A3: the odometry object's state (include/b2s.h "session state") ------------------------------------------------------------------
namespace b2s {
static_assert(sizeof(OdoState) % 8 == 0, "the state block is a section of whole words");

// the byte length of every section of an odometry blob (B2S_OS_*); returns the blob's total
static long long odometry_sections(long long buffer_size, long long n_prev, long long* len) {
  len[B2S_OS_PARAMS] = (sizeof(b2s_odometry_params) + 7) & ~(size_t)7;
  len[B2S_OS_MOTION] = (sizeof(b2s_motion_compensation_params) + 7) & ~(size_t)7;
  len[B2S_OS_STATE] = sizeof(OdoState);
  len[B2S_OS_RING_TIMES] = len[B2S_OS_MAP_TIMES] = 8 * buffer_size;
  len[B2S_OS_RING_POSES] = len[B2S_OS_MAP_POSES] = 128 * buffer_size;
  len[B2S_OS_PREV_XYZ] = len[B2S_OS_PREV_NORMALS] = 24 * n_prev;
  long long total = B2S_STATE_HEADER_BYTES;
  for (int k = 0; k < B2S_OS_COUNT; k++) total += len[k];
  return total;
}
}  // namespace b2s

extern "C" {

int32_t b2s_odometry_export_state(b2s_handle* h, const b2s_odometry* od, void* host_or_null, size_t capacity, size_t* n_bytes) {
  B2S_REQUIRE(h && od && n_bytes, B2S_E_INVALID, "null argument");
  B2S_REQUIRE(od->h == h, B2S_E_INVALID, "the odometry belongs to another handle");
  LOCK(h);
  int32_t n_prev = 0;   // synchronisation 1: the size of cloudPrev_
  B2S_TRY(read_back(h, {{&n_prev, od->prev->dn.p, 4}}));
  long long len[B2S_OS_COUNT];
  const long long bs = od->params.buffer_size;
  const long long total = odometry_sections(bs, n_prev, len);
  *n_bytes = (size_t)total;
  if (!host_or_null) return B2S_OK;
  B2S_REQUIRE((size_t)total <= capacity, B2S_E_CAPACITY, "the blob takes %lld bytes, the buffer holds %zu", total, capacity);
  unsigned char* b = static_cast<unsigned char*>(host_or_null);
  memset(b, 0, B2S_STATE_HEADER_BYTES);
  unsigned long long w[B2S_STATE_HEADER_BYTES / 8] = {0};
  w[B2S_STATE_W_MAGIC] = B2S_STATE_MAGIC_ODOMETRY; w[B2S_STATE_W_VERSION] = B2S_STATE_VERSION; w[B2S_STATE_W_BYTE_ORDER] = B2S_STATE_BYTE_ORDER;
  w[B2S_STATE_W_TOTAL_BYTES] = (unsigned long long)total;
  memcpy(&w[B2S_STATE_W_MAP_VOXEL], &h->cfg.map_voxel_size, 8);
  w[B2S_STATE_W_N_SECTIONS] = B2S_OS_COUNT;
  for (int k = 0; k < B2S_OS_COUNT; k++) w[B2S_STATE_W_SECTIONS + k] = (unsigned long long)len[k];
  w[B2S_OP_CAPACITY] = od->capacity; w[B2S_OP_BUFFER_SIZE] = (unsigned long long)bs; w[B2S_OP_N_PREV] = (unsigned long long)n_prev;
  w[B2S_OP_HOST_STEP] = (unsigned long long)od->host_step; w[B2S_OP_HAS_T] = od->has_t ? 1 : 0; w[B2S_OP_LAST_T] = (unsigned long long)od->last_t;
  memcpy(b, w, sizeof(w));
  long long off = B2S_STATE_HEADER_BYTES;
  unsigned char* sec[B2S_OS_COUNT];
  for (int k = 0; k < B2S_OS_COUNT; k++) { sec[k] = b + off; memset(sec[k], 0, (size_t)len[k]); off += len[k]; }
  memcpy(sec[B2S_OS_PARAMS], &od->params, sizeof(b2s_odometry_params));
  memcpy(sec[B2S_OS_MOTION], &od->mc, sizeof(b2s_motion_compensation_params));
  const std::pair<const DevBuf*, int> dev[] = {{&od->state, B2S_OS_STATE}, {&od->ring_t, B2S_OS_RING_TIMES}, {&od->ring_T, B2S_OS_RING_POSES},
                                               {&od->map_t, B2S_OS_MAP_TIMES}, {&od->map_T, B2S_OS_MAP_POSES}, {&od->prev->xyz, B2S_OS_PREV_XYZ},
                                               {&od->prev->nrm, B2S_OS_PREV_NORMALS}};
  for (const auto& d : dev)
    if (len[d.second]) B2S_CUDA(cudaMemcpyAsync(sec[d.second], d.first->p, (size_t)len[d.second], cudaMemcpyDeviceToHost, h->stream));
  return check_status(h);   // synchronisation 2: the data
}

int32_t b2s_odometry_import_state(b2s_handle* h, const void* blob, size_t n_bytes, b2s_odometry** out) {
  B2S_REQUIRE(h && blob && out, B2S_E_INVALID, "null argument");
  const unsigned char* b = static_cast<const unsigned char*>(blob);
  unsigned long long w[B2S_STATE_HEADER_BYTES / 8];
  B2S_REQUIRE(n_bytes >= B2S_STATE_HEADER_BYTES, B2S_E_INVALID, "state blob: %zu bytes, shorter than its header", n_bytes);
  memcpy(w, b, sizeof(w));
  B2S_REQUIRE(w[B2S_STATE_W_MAGIC] == B2S_STATE_MAGIC_ODOMETRY, B2S_E_INVALID, "state blob: not an odometry blob (magic)");
  B2S_REQUIRE(w[B2S_STATE_W_VERSION] == B2S_STATE_VERSION, B2S_E_INVALID, "state blob: format version %llu, this library reads %d",
              w[B2S_STATE_W_VERSION], B2S_STATE_VERSION);
  B2S_REQUIRE(w[B2S_STATE_W_BYTE_ORDER] == B2S_STATE_BYTE_ORDER, B2S_E_INVALID, "state blob: foreign byte order");
  B2S_REQUIRE(w[B2S_STATE_W_TOTAL_BYTES] == n_bytes, B2S_E_INVALID, "state blob: %zu bytes, its header says %llu", n_bytes, w[B2S_STATE_W_TOTAL_BYTES]);
  B2S_REQUIRE(w[B2S_STATE_W_N_SECTIONS] == B2S_OS_COUNT, B2S_E_INVALID, "state blob: %llu sections, an odometry blob has %d",
              w[B2S_STATE_W_N_SECTIONS], (int)B2S_OS_COUNT);
  const unsigned long long cap = w[B2S_OP_CAPACITY], bs = w[B2S_OP_BUFFER_SIZE], n_prev = w[B2S_OP_N_PREV];
  B2S_REQUIRE(cap >= 1 && cap < (unsigned long long)0x7fffffff / 4 && bs >= 1 && bs <= (1ull << 24) && n_prev <= cap, B2S_E_INVALID,
              "state blob: capacity %llu, buffer size %llu, %llu previous points", cap, bs, n_prev);
  long long len[B2S_OS_COUNT];
  const long long total = odometry_sections((long long)bs, (long long)n_prev, len);
  for (int k = 0; k < B2S_OS_COUNT; k++)
    B2S_REQUIRE(w[B2S_STATE_W_SECTIONS + k] == (unsigned long long)len[k], B2S_E_INVALID, "state blob: section %d holds %llu bytes, its counts give %lld",
                k, w[B2S_STATE_W_SECTIONS + k], len[k]);
  B2S_REQUIRE((unsigned long long)total == n_bytes, B2S_E_INVALID, "state blob: sections of %lld bytes in %zu", total, n_bytes);
  const unsigned char* sec[B2S_OS_COUNT];
  long long off = B2S_STATE_HEADER_BYTES;
  for (int k = 0; k < B2S_OS_COUNT; k++) { sec[k] = b + off; off += len[k]; }
  b2s_odometry_params p;
  b2s_motion_compensation_params mc;
  OdoState s;
  memcpy(&p, sec[B2S_OS_PARAMS], sizeof(p));
  memcpy(&mc, sec[B2S_OS_MOTION], sizeof(mc));
  memcpy(&s, sec[B2S_OS_STATE], sizeof(s));
  B2S_TRY(check_odometry_params(p));
  B2S_REQUIRE((unsigned long long)p.buffer_size == bs, B2S_E_INVALID, "state blob: buffer size %d, the header says %llu", (int)p.buffer_size, bs);
  B2S_REQUIRE(mc.scan_duration > 0.0 && mc.num_poses_velocity_estimation >= 1, B2S_E_INVALID, "state blob: de-skew parameters");
  const long long B = (long long)bs;
  B2S_REQUIRE(s.head >= 0 && s.head < B && s.count >= 0 && s.count <= B && s.map_head >= 0 && s.map_head < B && s.map_count >= 0 &&
                  s.map_count <= B && s.slot >= 0 && s.slot < 256, B2S_E_INVALID, "state blob: a buffer position or result slot out of range");
  LOCK(h);
  return create_object(out, [&](b2s_odometry* od) -> int32_t {
    B2S_TRY(odometry_init(h, od, &p, (size_t)cap));
    if (mc.enabled) B2S_TRY(odometry_deskew_buffers(h, od));
    memcpy(&od->params, sec[B2S_OS_PARAMS], sizeof(b2s_odometry_params));   // byte for byte, padding included: a re-export is identical
    memcpy(&od->mc, sec[B2S_OS_MOTION], sizeof(b2s_motion_compensation_params));
    const std::pair<DevBuf*, int> dev[] = {{&od->state, B2S_OS_STATE}, {&od->ring_t, B2S_OS_RING_TIMES}, {&od->ring_T, B2S_OS_RING_POSES},
                                           {&od->map_t, B2S_OS_MAP_TIMES}, {&od->map_T, B2S_OS_MAP_POSES}, {&od->prev->xyz, B2S_OS_PREV_XYZ},
                                           {&od->prev->nrm, B2S_OS_PREV_NORMALS}};
    for (const auto& d : dev)
      if (len[d.second]) B2S_CUDA(cudaMemcpyAsync(d.first->p, sec[d.second], (size_t)len[d.second], cudaMemcpyHostToDevice, h->stream));
    B2S_TRY(cloud_set_count(h, od->prev.get(), (size_t)n_prev));
    od->host_step = (long long)w[B2S_OP_HOST_STEP];
    od->has_t = w[B2S_OP_HAS_T] != 0;
    od->last_t = (long long)w[B2S_OP_LAST_T];
    return check_status(h);
  });
}

}  // extern "C"
