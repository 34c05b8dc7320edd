// Per-object code: state initialisation (+ work-queue seeding), normal-equation assembly from the tile partials,
// register-resident elimination, Sim(3)/SE(3) update (kernel k_solve and device function solve_object),
// and the per-ray occupancy scan / band compaction of the render term.
// Restates optimizer.py:45-86, 97-203; loss.py:84-141, 155-178; loss_utils.py:188-233.
#pragma once
#include "dspgn_common.cuh"
#include "dspgn_simt.cuh"

namespace dspgn {

template <class T>
__device__ __forceinline__ T ldv(const T* p) { return *reinterpret_cast<const volatile T*>(p); }

// ---- multi-GPU result exchange (GatherDev: dspgn_common.cuh) ------------------------------------------------
__device__ __forceinline__ int ld_acquire_sys(const int* p) {
  int v;
  asm volatile("ld.acquire.sys.global.s32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_release_sys(int* p, int v) {
  asm volatile("st.release.sys.global.s32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ unsigned long long globaltimer_ns() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}
constexpr unsigned long long kPeerTimeoutNs = 20ull * 1000ull * 1000ull * 1000ull;   // soft failure, never a trap

// spin until *p >= need (system scope); false on timeout
__device__ inline bool wait_ge_sys(const int* p, int need) {
  const unsigned long long t0 = globaltimer_ns();
  while (ld_acquire_sys(p) < need) {
    __nanosleep(200);
    if (globaltimer_ns() - t0 > kPeerTimeoutNs) return false;
  }
  return true;
}

// flow control at the start of a step: rank 0 acknowledges everything before the previous step as consumed (its
// stream ran the D2H / consumers of step seq-2 before this kernel); the others make sure the slot set they are
// about to overwrite (written two steps ago) has been consumed.
__device__ inline void gather_step_begin(const GatherDev& g) {
  if (g.slots == nullptr) return;
  if (g.rank == 0) st_release_sys(g.ack, g.seq - 1);
  else if (!wait_ge_sys(g.ack, g.seq - 2)) *g.err = 1;
}

// end of a step (its own launch, stream-ordered behind every kernel that stored records): publish
__global__ void k_gather_publish(GatherDev g, int with_begin) {
  if (threadIdx.x != 0) return;
  if (with_begin) gather_step_begin(g);          // rank without objects this step: no k_init ran
  __threadfence_system();
  st_release_sys(g.flags + g.rank, g.seq);
}

// rank 0: wait until every rank has published step seq
__global__ void k_gather_wait(GatherDev g) {
  const int r = threadIdx.x;
  const unsigned long long t0 = globaltimer_ns();
  bool ok = true;
  if (r < g.world) ok = wait_ge_sys(g.flags + r, g.seq);
  if (!ok) *g.err = 1;
  __syncwarp();
  if (r == 0) *g.wait_ns = (long long)(globaltimer_ns() - t0);
}

// Result record of one object (DspgnObjectOut layout): pose back in camera<-object form (optimizer.py:200 / :83-84),
// code, loss, status, counters; mirrored into rank 0's gather buffer when the exchange is on.
__device__ inline void write_record(float* results, const GatherDev& g, int o, const ObjState& st, float scale) {
  float* r = results + (size_t)o * DSPGN_RESULT_FLOATS;
  float Toc[12], Tco[12];
  for (int i = 0; i < 12; ++i) Toc[i] = ldv(&st.T_oc[i]);
  inv_affine(Toc, Tco, nullptr);                         // optimizer.py:200 / :83
  if (st.mode == DSPGN_MODE_POSE) {                      // optimizer.py:84: t_cam_obj[:3,:3] /= scale
    for (int i = 0; i < 3; ++i)
      for (int c = 0; c < 3; ++c) Tco[i * 4 + c] /= scale;
  }
  for (int i = 0; i < 12; ++i) r[i] = Tco[i];
  r[12] = 0.f; r[13] = 0.f; r[14] = 0.f; r[15] = 1.f;
  for (int i = 0; i < kMaxCode; ++i) r[16 + i] = ldv(&st.z[i]);
  r[80] = ldv(&st.loss);
  reinterpret_cast<int*>(r)[81] = ldv(&st.status);
  reinterpret_cast<int*>(r)[82] = ldv(&st.V);
  reinterpret_cast<int*>(r)[83] = ldv(&st.m);
  reinterpret_cast<int*>(r)[84] = ldv(&st.iters);
  reinterpret_cast<int*>(r)[85] = 0;
  reinterpret_cast<int*>(r)[86] = 0;
  reinterpret_cast<int*>(r)[87] = 0;
  if (g.slots != nullptr) {
    // multi-GPU: the same record into the object's slot of rank 0's gather buffer.  On ranks > 0 this is a
    // peer-mapped address: plain st.global that travel over NVLink; they are published by k_gather_publish.
    float4* dst = reinterpret_cast<float4*>(g.slots + (size_t)g.slot_of[o] * DSPGN_RESULT_FLOATS);
    const float4* src = reinterpret_cast<const float4*>(r);
#pragma unroll 2
    for (int i = 0; i < DSPGN_RESULT_FLOATS / 4; ++i) dst[i] = src[i];
  }
}

// ---- the map-consistency check of a tracked detection (dspgn_keyframe_batch_gated) -----------------------------------
// GetNewObservations (src/LocalMapping_util.cc:104-147) compares the pose-only estimate Zco with the pose the map
// predicts, Tco = Tcw Two: dist2D, the x/z translation difference in fp32 (Eigen::Vector2f::norm), and e = log(Tco^-1 Zco)
// with both poses as g2o SE3Quat (unit quaternion + translation, fp64).  Restated here:
//   quaternion of a rotation matrix: the trace form when tr > 0, else the form pivoted on the largest diagonal entry;
//   then the sign is chosen so that w >= 0 and the quaternion is normalised (SE3Quat(R, t));
//   inverse (q*, -q* t), product (t1 + q1 t2, q1 q2, renormalised);
//   log: R of the quaternion, d = (tr R - 1) / 2, dR = (R21 - R12, R02 - R20, R10 - R01);
//        d > 0.99999:  w = dR / 2,                                V^-1 = I - W/2 + W^2/12
//        otherwise:    w = acos(d) / (2 sqrt(1 - d^2)) dR,      V^-1 = I - W/2 + (1 - th / (2 tan(th/2))) / th^2 W^2
//        u = V^-1 t,  e = (w, u).
// Kept: dist2D < 1 and |e| < 1.5 (a NaN fails).  oracle/gate_check.py is the same check in numpy.
struct GateQuat { double w, x, y, z; };
__device__ inline GateQuat gate_normalise(GateQuat q) {
  if (q.w < 0.0) { q.w = -q.w; q.x = -q.x; q.y = -q.y; q.z = -q.z; }
  const double n = sqrt(q.w * q.w + q.x * q.x + q.y * q.y + q.z * q.z);
  q.w /= n; q.x /= n; q.y /= n; q.z /= n;
  return q;
}
// rotation part of a row-major 4x4 float matrix (fp64), normalised quaternion
__device__ inline GateQuat gate_quat(const float* T) {
  double m[3][3];
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 3; ++c) m[r][c] = (double)T[r * 4 + c];
  double v[4];                                       // x, y, z, w
  const double tr = m[0][0] + m[1][1] + m[2][2];
  if (tr > 0.0) {
    const double s = sqrt(tr + 1.0), h = 0.5 / s;
    v[3] = 0.5 * s;
    v[0] = (m[2][1] - m[1][2]) * h; v[1] = (m[0][2] - m[2][0]) * h; v[2] = (m[1][0] - m[0][1]) * h;
  } else {
    int i = 0;
    if (m[1][1] > m[0][0]) i = 1;
    if (m[2][2] > m[i][i]) i = 2;
    const int j = (i + 1) % 3, k = (j + 1) % 3;
    const double s = sqrt(m[i][i] - m[j][j] - m[k][k] + 1.0), h = 0.5 / s;
    v[i] = 0.5 * s;
    v[3] = (m[k][j] - m[j][k]) * h;
    v[j] = (m[j][i] + m[i][j]) * h;
    v[k] = (m[k][i] + m[i][k]) * h;
  }
  return gate_normalise(GateQuat{v[3], v[0], v[1], v[2]});
}
__device__ inline GateQuat gate_qmul(const GateQuat& a, const GateQuat& b) {
  return GateQuat{a.w * b.w - a.x * b.x - a.y * b.y - a.z * b.z, a.w * b.x + a.x * b.w + a.y * b.z - a.z * b.y,
                  a.w * b.y - a.x * b.z + a.y * b.w + a.z * b.x, a.w * b.z + a.x * b.y - a.y * b.x + a.z * b.w};
}
// R of a unit quaternion, row-major
__device__ inline void gate_rot(const GateQuat& q, double R[9]) {
  const double tx = 2.0 * q.x, ty = 2.0 * q.y, tz = 2.0 * q.z;
  const double twx = tx * q.w, twy = ty * q.w, twz = tz * q.w, txx = tx * q.x, txy = ty * q.x, txz = tz * q.x;
  const double tyy = ty * q.y, tyz = tz * q.y, tzz = tz * q.z;
  R[0] = 1.0 - (tyy + tzz); R[1] = txy - twz;         R[2] = txz + twy;
  R[3] = txy + twz;         R[4] = 1.0 - (txx + tzz); R[5] = tyz - twx;
  R[6] = txz - twy;         R[7] = tyz + twx;         R[8] = 1.0 - (txx + tyy);
}
__device__ inline void gate_qrot(const GateQuat& q, const double v[3], double out[3]) {
  double R[9];
  gate_rot(q, R);
  for (int r = 0; r < 3; ++r) out[r] = R[3 * r] * v[0] + R[3 * r + 1] * v[1] + R[3 * r + 2] * v[2];
}
// DSPGN_GATE_KEPT or DSPGN_GATE_REJECTED for the estimate Z against the map's prediction M (row-major 4x4 floats)
__device__ __noinline__ int gate_decide(const float* Z, const float* M) {
  const float dx = __fsub_rn(Z[3], M[3]), dz = __fsub_rn(Z[11], M[11]);
  const float dist2d = sqrtf(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dz, dz)));
  const GateQuat qm = gate_quat(M), qz = gate_quat(Z);
  // Tco^-1 = (q*, -(q* t)),  Tco^-1 Zco = (q* tz + t_inv, q* qz)
  const GateQuat qi{qm.w, -qm.x, -qm.y, -qm.z};
  const double tm[3] = {-(double)M[3], -(double)M[7], -(double)M[11]}, tz[3] = {(double)Z[3], (double)Z[7], (double)Z[11]};
  double ti[3], tr[3];
  gate_qrot(qi, tm, ti);
  gate_qrot(qi, tz, tr);
  for (int i = 0; i < 3; ++i) tr[i] += ti[i];
  const GateQuat q = gate_normalise(gate_qmul(qi, qz));
  double R[9];
  gate_rot(q, R);
  const double d = 0.5 * (R[0] + R[4] + R[8] - 1.0);
  const double dR[3] = {R[7] - R[5], R[2] - R[6], R[3] - R[1]};
  double w[3], c2;
  if (d > 0.99999) {
    for (int i = 0; i < 3; ++i) w[i] = 0.5 * dR[i];
    c2 = 1.0 / 12.0;
  } else {
    const double th = acos(d), f = th / (2.0 * sqrt(1.0 - d * d));
    for (int i = 0; i < 3; ++i) w[i] = f * dR[i];
    c2 = (1.0 - th / (2.0 * tan(th / 2.0))) / (th * th);
  }
  // V^-1 t = t - W t / 2 + c2 W (W t),  W t = w x t
  const double wt[3] = {w[1] * tr[2] - w[2] * tr[1], w[2] * tr[0] - w[0] * tr[2], w[0] * tr[1] - w[1] * tr[0]};
  const double wwt[3] = {w[1] * wt[2] - w[2] * wt[1], w[2] * wt[0] - w[0] * wt[2], w[0] * wt[1] - w[1] * wt[0]};
  double e2 = 0.0;
  for (int i = 0; i < 3; ++i) {
    const double u = tr[i] - 0.5 * wt[i] + c2 * wwt[i];
    e2 += w[i] * w[i] + u * u;
  }
  return (dist2d < 1.0f && sqrt(e2) < 1.5) ? DSPGN_GATE_KEPT : DSPGN_GATE_REJECTED;
}

// Gate of a finished gated pose-only object o (one thread, after its record was written): the record's pose, or after a
// soft failure the input pose, against the map's prediction; the verdict goes into the record's gate word.
__device__ inline int gate_record(float* results, int o, const float* T_init, const float* t_map) {
  float* r = results + (size_t)o * DSPGN_RESULT_FLOATS;
  const float* Z = (reinterpret_cast<const int*>(r)[81] == DSPGN_ST_OK) ? r : T_init + 16 * (size_t)o;
  const int g = gate_decide(Z, t_map + 16 * (size_t)o);
  reinterpret_cast<int*>(r)[85] = g;
  return g;
}

// ---- cooperative stop (dspgn_keyframe_stop) -----------------------------------------------------------------------
// The stop word lives in pinned host memory: a system-scope load sees a host store (or another CTA's) without a fence.
__device__ __forceinline__ bool stop_seen(const StopDev& s) {
  unsigned v;
  asm volatile("ld.relaxed.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(s.word) : "memory");
  return v == s.gen;
}

// The solve of resident object o at iteration `iter` (one thread, beside the elimination): the test hook raises the stop,
// then a stoppable object's solve that is not its last reads the word.  1: the object stops after this iteration's
// update (unless the solve fails).
__device__ __forceinline__ int stop_check(const StopDev& s, int o, int iter, bool pose_only, bool last_iter) {
  if (s.word == nullptr) return 0;
  const bool can = !pose_only && !last_iter && (s.pair == nullptr || s.pair[o] < 0);
  if (o == s.dbg_obj && iter == s.dbg_iter && (can || pose_only))
    asm volatile("st.relaxed.sys.global.u32 [%0], %1;" :: "l"(s.word), "r"(s.gen) : "memory");
  return (can && stop_seen(s)) ? 1 : 0;
}

// The record of a rejected gated object's joint slot that a stop keeps from waking: its input pose (t_cam_obj_sim3), zero
// code, no iteration.  One thread.
__device__ inline void stopped_slot_record(float* results, ObjState* state, const float* T_init, int slot) {
  float* r = results + (size_t)slot * DSPGN_RESULT_FLOATS;
  for (int i = 0; i < 16; ++i) r[i] = T_init[16 * (size_t)slot + i];
  for (int i = 16; i < DSPGN_RESULT_FLOATS; ++i) r[i] = 0.f;
  reinterpret_cast<int*>(r)[81] = DSPGN_ST_STOPPED;
  state[slot].status = DSPGN_ST_STOPPED;
}

// ---- device-side input construction (SURVEY 8 row f4) --------------------------------------------------------------
// Runs once per upload, in place on the uploaded staging block: ray slots hold (u, v, 1) and become inv_k [u, v, 1]
// (loss_utils.py:23-37 / LocalMapping_util.cc:378-386); world map points become camera points x_c = R x_w + t
// (LocalMapping_util.cc:344-352) and the object's world pose is composed with the camera pose, T_co = T_cw T_wo (:390).
// aux[o]: inv_k (9, row-major) | T_cw (12, rows of [R|t]).
struct BuildArgs { const ObjMeta* meta; float* T_init; float* pts; float* rays; const float* aux; int n_obj; };
constexpr int kAuxFloats = 24;
__global__ void k_build_inputs(BuildArgs a) {
  const int o = blockIdx.x, tid = threadIdx.x;
  const ObjMeta M = a.meta[o];
  if (M.build == 0) return;
  const float* ax = a.aux + (size_t)o * kAuxFloats;
  if (M.build & 1) {
    float K[9];
#pragma unroll
    for (int i = 0; i < 9; ++i) K[i] = ax[i];
    for (int i = tid; i < M.n_rays; i += blockDim.x) {
      float* r = a.rays + 3 * (size_t)(M.ray_off + i);
      const float u = r[0], v = r[1];
#pragma unroll
      for (int k = 0; k < 3; ++k) r[k] = __fadd_rn(__fmaf_rn(K[3 * k + 1], v, __fmul_rn(K[3 * k], u)), K[3 * k + 2]);
    }
  }
  if (M.build & 2) {
    float T[12];
#pragma unroll
    for (int i = 0; i < 12; ++i) T[i] = ax[9 + i];
    for (int i = tid; i < M.n_pts; i += blockDim.x) {
      float* p = a.pts + 3 * (size_t)(M.pts_off + i);
      float x, y, z;
      xform_point(T, p[0], p[1], p[2], x, y, z);
      p[0] = x; p[1] = y; p[2] = z;
    }
    if (tid == 0) {
      float* Tw = a.T_init + 16 * (size_t)o;
      float B[12], C[12];
      for (int i = 0; i < 12; ++i) B[i] = Tw[i];
      mul_affine(T, B, C);
      for (int i = 0; i < 12; ++i) Tw[i] = C[i];
    }
  }
}

// ---- valid-sample ranges of the rays (persistent kernel with the render term) ------------------------------------------
// loss.py:68 keeps the ray samples inside the unit sphere (the reference decodes only those V samples, loss.py:77-78).
// Along a ray they are one run of consecutive samples (a line meets a ball in a segment) -- 70 % of the n_rays * D samples
// on the real SLAM shape, 80-93 % on the BASELINE configs -- so the forward-only tiles of the persistent kernel enumerate
// only the hull [first valid, last valid] of every ray:
//   vpre[ray] = (exclusive prefix of the hull lengths << kRangeSampleBits) | first valid sample,
//   vpre[n_rays] = total << kRangeSampleBits.
// Sample positions and the inside test are the tile prologue's own (lin_depth, xform_point, inside_unit_sphere), so a hull
// contains exactly the samples the full enumeration marks valid; the prologue still tests every row it is given.
// Only the samples next to the two ends of a hull are actually tested: the chord of the ray inside the unit ball
// (|u d + t| < 1 with u = R_oc q) brackets the hull to within a fraction of a sample, the search window is that bracket
// +- 2 samples, found ends are extended outwards while the neighbour is valid, and a ray with an empty window is scanned
// completely unless its line misses the ball by more than 1 % of the radius -- so the result is the hull of the exhaustive
// test of all D samples (tests/valid_ranges_model.py checks the window against it).
// Called by all `nthreads` (multiple of 32, <= 1024) threads; s_wsum: 32 ints of shared memory.  Returns the total.
__device__ __forceinline__ int vpre_base(const ObjMeta& M, int o) { return M.ray_off + o; }
template <bool NAMED_BAR>
__device__ __forceinline__ void vpre_sync() {
  if (NAMED_BAR) asm volatile("bar.sync 1, 256;" ::: "memory");
  else __syncthreads();
}
template <bool NAMED_BAR>
__device__ inline int valid_sample_ranges(const ObjMeta& M, const ObjState& st, const float* __restrict__ rays, const int D,
                                          int* vp, const int tid, const int nthreads, int* s_wsum) {
  const int lane = tid & 31, warp = tid >> 5, nw = nthreads >> 5;
  float T[12];
#pragma unroll
  for (int i = 0; i < 12; ++i) T[i] = ldv(&st.T_oc[i]);
  const float dmin = ldv(&st.dmin), dmax = ldv(&st.dmax), dstep = ldv(&st.dstep);
  int carry = 0;
  for (int r0 = 0; r0 < M.n_rays; r0 += nthreads) {
    const int ray = r0 + tid;
    int first = 0, cnt = 0;
    if (ray < M.n_rays) {
      const float* q = rays + 3 * (size_t)(M.ray_off + ray);
      const float q0 = q[0], q1 = q[1], q2 = q[2];
      auto valid = [&](int j) -> bool {           // exactly the tile prologue's test of sample j
        const float d = lin_depth(dmin, dmax, dstep, j, D);
        float x, y, z;
        xform_point(T, __fmul_rn(q0, d), __fmul_rn(q1, d), __fmul_rn(q2, d), x, y, z);
        return inside_unit_sphere(x, y, z);
      };
      int w0 = 0, w1 = D - 1;                     // search window (inclusive)
      bool none = false;
      const float ux = T[0] * q0 + T[1] * q1 + T[2] * q2, uy = T[4] * q0 + T[5] * q1 + T[6] * q2, uz = T[8] * q0 + T[9] * q1 + T[10] * q2;
      const float aa = ux * ux + uy * uy + uz * uz, bb = ux * T[3] + uy * T[7] + uz * T[11];
      const float cc = T[3] * T[3] + T[7] * T[7] + T[11] * T[11] - 1.0f;
      if (aa > 1e-20f && aa < 1e20f && dstep > 1e-12f && fabsf(dmin) < 1e4f && fabsf(dmax) < 1e4f && fabsf(bb) < 1e20f && fabsf(cc) < 1e20f) {
        const float inv = 1.0f / aa;
        if (cc - bb * bb * inv > 0.02f) none = true;          // closest approach > 1.01: no sample can test inside
        else {
          const float sq = sqrtf(fmaxf(bb * bb - aa * cc, 0.f)) * inv, dc = -bb * inv;
          const float flo = (dc - sq - dmin) / dstep, fhi = (dc + sq - dmin) / dstep;      // chord ends in sample units
          if (flo == flo && fhi == fhi) {                      // (NaN: keep the full window)
            if (fhi < -2.0f || flo > (float)(D + 1)) none = true;   // the chord ends two samples before the first / starts two after the last
            else {
              w0 = max(0, (int)floorf(fmaxf(flo, -4.0f)) - 2);
              w1 = min(D - 1, (int)ceilf(fminf(fhi, (float)(D + 4))) + 2);
            }
          }
        }
      }
      int lo = -1, hi = -1;
      if (!none) {
        for (int j = w0; j <= w1; ++j) if (valid(j)) { lo = j; break; }
        if (lo < 0 && (w0 > 0 || w1 < D - 1)) {                 // nothing next to the chord (not expected): test every sample
          w1 = D - 1;
          for (int j = 0; j < D; ++j) if (valid(j)) { lo = j; break; }
        }
        if (lo >= 0) {
          while (lo > 0 && valid(lo - 1)) --lo;
          hi = lo;
          for (int j = w1; j > lo; --j) if (valid(j)) { hi = j; break; }
          while (hi < D - 1 && valid(hi + 1)) ++hi;
        }
      }
      if (lo >= 0) { first = lo; cnt = hi - lo + 1; }
    }
    int x = cnt;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) { const int y = __shfl_up_sync(0xffffffffu, x, d); if (lane >= d) x += y; }
    if (lane == 31) s_wsum[warp] = x;
    vpre_sync<NAMED_BAR>();
    int woff = 0, tot = 0;
    for (int w = 0; w < nw; ++w) { const int v = s_wsum[w]; if (w < warp) woff += v; tot += v; }
    if (ray < M.n_rays) vp[ray] = ((carry + woff + x - cnt) << kRangeSampleBits) | first;
    carry += tot;
    vpre_sync<NAMED_BAR>();
  }
  if (tid == 0) vp[M.n_rays] = carry << kRangeSampleBits;
  return carry;
}

struct InitArgs {
  int code_len;
  int n_iter_joint, n_iter_pose;   // GN iterations of a joint / pose-only object
  int n_bad;                       // objects rejected at upload (they count as done from the start)
  int tile_rows;                   // rows per tile of the persistent kernel that runs next (its iteration-0 items)
};

// zb0 = b0 + W0[:, :L] z   (fp32 FMA chain in i order; all threads of the calling CTA / epilogue)
__device__ __forceinline__ void refresh_zb0(ObjState& st, const DecoderDev& dec, int tid, int nthreads) {
  const float* __restrict__ W = dec.Wf[0];      // reduction-major [in][256]
  const float* __restrict__ b = dec.bias[0];
  for (int j = tid; j < kHid; j += nthreads) {
    float acc = b[j];
    for (int i = 0; i < dec.L; ++i) acc = fmaf(W[i * kHid + j], ldv(&st.z[i]), acc);
    st.zb0[j] = acc;
  }
}

// q.q_flag != nullptr: the persistent kernel runs next, so also seed its work queue with every object's iteration-0
// tiles (ray-sample tiles first)
__global__ void k_init(BatchDev b, InitArgs a, MegaArgs q) {
  const int o = blockIdx.x, tid = threadIdx.x;
  const bool mega = q.q_flag != nullptr;
  if (o == 0 && tid == 0) gather_step_begin(b.gather);
  ObjState& st = b.state[o];
  const ObjMeta M = b.meta[o];
  const int mode = b.modes[o];
  const int link = (b.link != nullptr) ? b.link[o] : -1;
  // the joint slot of a gated object starts dormant: fully initialised here, no tiles queued; the solve step that finishes
  // its pose-only object wakes it (persistent kernel) or k_gate_wake does (per-iteration schedule, n_iter 0 until then)
  const bool dormant = link >= 0 && mode == DSPGN_MODE_JOINT;
  if (tid < kMaxCode) st.z[tid] = (M.has_code && tid < a.code_len) ? b.code_init[o * kMaxCode + tid] : 0.f;
  if (tid == 0) {
    float Tco[12];
    for (int r = 0; r < 3; ++r)
      for (int c = 0; c < 4; ++c) Tco[r * 4 + c] = b.T_init[o * 16 + r * 4 + c];
    if (mode == DSPGN_MODE_POSE)           // optimizer.py:54: t_cam_obj[:3,:3] *= scale
      for (int r = 0; r < 3; ++r)
        for (int c = 0; c < 3; ++c) Tco[r * 4 + c] *= M.scale;
    inv_affine(Tco, st.T_oc, nullptr);     // optimizer.py:55 / :104
    derive_depth_range(st, b.D);
    st.loss = 0.f; st.status = M.bad ? DSPGN_ST_BAD_INPUT : 0; st.iters = 0; st.V = 0; st.m = 0; st.n_active = M.n_pts;
    st.mode = mode; st.n_iter = (mode == DSPGN_MODE_POSE) ? a.n_iter_pose : ((dormant && !mega) ? 0 : a.n_iter_joint);
    b.V_count[o] = 0;
    b.band_m[o] = 0;
  }
  __syncthreads();
  refresh_zb0(st, b.decs[M.class_id], tid, blockDim.x);
  if (M.bad) {                               // rejected at upload: no tile, no solve -- its record is final now
    __syncthreads();
    if (tid == 0) write_record(b.results, b.gather, o, st, M.scale);
    // a gated object rejected at upload is checked with its input pose; its joint slot has the same points, rays and
    // depths, so it is rejected at upload too and its record is already final
    if (tid == 0 && link >= 0 && mode == DSPGN_MODE_POSE) gate_record(b.results, o, b.T_init, b.t_map);
  }
  if (mega) {
    const int rows = a.tile_rows;
    const int ntS = (M.n_pts + rows - 1) / rows;
    // slots reserved by the host for this object's iteration 0: every ray sample (joint objects of a run with the render
    // term) + every SDF tile
    const int ntF_cap = (q.render && !M.bad && mode == DSPGN_MODE_JOINT) ? (M.n_rays * b.D + rows - 1) / rows : 0;
    int ntF = ntF_cap;
    if (q.vpre != nullptr && ntF_cap > 0) {
      __shared__ int s_wsum[32];
      __syncthreads();                         // T_oc / depth range written by thread 0 above
      const int vh = valid_sample_ranges<false>(M, st, b.rays, b.D, q.vpre + vpre_base(M, o), tid, blockDim.x, s_wsum);
      ntF = (vh + rows - 1) / rows;
    }
    const int base = b.q0_off[o];
    if (!dormant) {                          // a dormant slot has no reserved slots: its wake pushes these items
      for (int j = tid; j < ntF; j += blockDim.x) q.q_flag[base + j] = make_item(MODE_RAYFWD, o, j) + 1;
      for (int j = tid; j < ntS; j += blockDim.x) q.q_flag[base + ntF + j] = make_item(MODE_SDF, o, j) + 1;
      for (int j = ntF + ntS + tid; j < ntF_cap + ntS; j += blockDim.x) q.q_flag[base + j] = kItemNop + 1;
    }
    if (tid == 0) { q.pending[o] = ntS + (ntF > 0 ? 1 : 0); q.ray_left[o] = ntF; q.obj_iter[o] = 0; }
    if (o == 0 && tid == 0) {
      QueueCounters& c = *q.ctr;
      c.head = 0; c.tail = q.total0; c.done_objects = a.n_bad; c.band_rows_total = 0; c.valid_rows_total = 0ull; c.abort_flag = 0;
    }
  }
}

// ---------------------------------------------------------------------------------------------
struct SolveArgs {
  const float* part_s;     // SDF-term tile partials [tile][kAccStride]
  const float* part_r;     // render-term (band rows) tile partials
  const int* base_s;       // [n_obj] first tile of each object in the SDF / band launches
  const int* base_r;
  int tile_rows;           // rows per tile of the decoder engine
  SolverParams prm;
  int iter_index;         // per-iteration schedule: the iteration being solved (an object's last one writes its record)
  // debug: dump the system of object dbg_obj and do not update any state
  int dbg_obj; float* dbg_H; float* dbg_b; float* dbg_dx; float* dbg_loss;
};

constexpr int kSolveThreads = 256;
constexpr int kPMax = 7 + kMaxCode;   // 71
constexpr int kAsStride = kPMax + 2;  // 73 floats: odd stride -> thread-per-row reads are bank-conflict free
constexpr int kMaxEnt = (kTriInt + kPInt + kSolveThreads - 1) / kSolveThreads;   // 11 entries of a tile partial per thread

__device__ __forceinline__ int ext_to_int(int e, int npose, int L) {
  // external order [pose | code]  ->  internal rows [code 0..63 | pose 64..70]
  return (e < npose) ? (kMaxCode + e) : (e - npose);
}

// BatchDev::lin: floats per slot at code length L, and entry (r, c), r <= c, of a slot's P x P system (external order)
__host__ __device__ __forceinline__ int lin_floats(int L) { return (7 + L) * (8 + L) / 2; }
__host__ __device__ __forceinline__ int lin_index(int r, int c, int P) { return r * P - (r * (r - 1)) / 2 + (c - r); }

__device__ __forceinline__ void write_result(const BatchDev& b, int o, const ObjState& st) {
  write_record(b.results, b.gather, o, st, b.meta[o].scale);
}

constexpr int kElimThreads = 96;      // rows 0..70 live in the first three warps
__device__ __forceinline__ void elim_bar() { asm volatile("bar.sync 2, 96;" ::: "memory"); }

// Shared-memory workspace of one solve (static in k_solve, carved from the J tile in the persistent kernel)
struct SolveSmem {
  float As[kPMax * kAsStride];                 // assembled augmented system [H | b]
  float4 bcast[2][(kPMax + 1) / 4 + 1];        // pivot row + rhs broadcast (double buffered)
  float xs[kPMax];
  float s_rot[4];                              // J_rot.x, J_rot.z, res_rot, active
  double s_sum[4];                             // sdf loss sum, sdf rows, render loss sum
  int s_flag;
  int s_stop;                                  // the object observed a stop at the end of this solve
};

// MEGA = called by the 256 epilogue threads of the persistent decoder kernel (named barrier, other CTAs wrote
// the data: cache-bypassing loads); otherwise by the 256 threads of k_solve.
template <bool MEGA>
__device__ __forceinline__ void solve_sync() {
  if (MEGA) asm volatile("bar.sync 1, 256;" ::: "memory");
  else __syncthreads();
}

// Pivots [k0, k1) of the register-resident Gauss-Jordan elimination, touching the first 4*NCH entries of the rotated
// rows (all later entries are zero on entry and stay zero).  Called by threads 0..95; one named barrier per pivot.
template <int NCH>
__device__ __forceinline__ void gj_pivots(const int k0, const int k1, const int tid, float (&arow)[kPMax + 1], float& brow,
                                          float& mydiag, int& bad_pivot, float4 (&bcast)[2][(kPMax + 1) / 4 + 1]) {
  constexpr int NE = 4 * NCH;                      // entries 0 .. NE-1 are live (entry NE-1 is already zero)
#pragma unroll 1
  for (int k = k0; k < k1; ++k) {
    float4* buf = bcast[k & 1];
    if (tid == k) {
#pragma unroll
      for (int j = 0; j < NE; j += 4) buf[j >> 2] = make_float4(arow[j], arow[j + 1], arow[j + 2], arow[j + 3]);
      buf[(kPMax + 1) / 4] = make_float4(brow, 0.f, 0.f, 0.f);
      mydiag = arow[0];
    }
    elim_bar();
    float pr[NE];
#pragma unroll
    for (int j = 0; j < NE; j += 4) {
      const float4 v = buf[j >> 2];
      pr[j] = v.x; pr[j + 1] = v.y; pr[j + 2] = v.z; pr[j + 3] = v.w;
    }
    const float pb = buf[(kPMax + 1) / 4].x;
    const float piv = pr[0];
    if (!(piv > 0.f) || !(piv < 3.0e38f)) bad_pivot = 1;        // every thread sees the same pivot
    const float l = (tid == k) ? 0.f : __fdividef(arow[0], piv);        // MUFU.RCP path, shorter than __frcp_rn (tools/probes/solve_probe.cu)
#pragma unroll
    for (int j = 1; j < NE; ++j) arow[j - 1] = fmaf(-l, pr[j], arow[j]);
    brow = fmaf(-l, pb, brow);
  }
}

// One CTA (or the epilogue half of one) per object: fixed-order reduction of the tile partials (fp64), priors
// and damping (optimizer.py:161-184), Gauss-Jordan elimination of the SPD 71x71 system with thread = row in
// registers (the system ends diagonal: no back-substitution), Sim(3)/SE(3) update, next depth range, soft failures
// (optimizer.py:130-150).  `log`: the persistent kernel's event log (solve phases).
// Returns 1 when the object is finished (last iteration, frozen or soft-failed), else 0.
template <bool MEGA>
__device__ int solve_object(const BatchDev& b, const SolveArgs& a, const EventLog& log, const int o, const int tid, SolveSmem& SM,
                            const bool last_iter) {
  float (&As)[kPMax * kAsStride] = SM.As;
  float4 (&bcast)[2][(kPMax + 1) / 4 + 1] = SM.bcast;
  float (&xs)[kPMax] = SM.xs;
  float (&s_rot)[4] = SM.s_rot; double (&s_sum)[4] = SM.s_sum; int& s_flag = SM.s_flag;
  ObjState& st = b.state[o];
  const SolverParams& prm = a.prm;
  const int L = prm.code_len;
  const bool pose_only = st.mode == DSPGN_MODE_POSE;      // estimate_pose_cam_obj variant
  const int npose = pose_only ? 6 : 7;
  const int P = pose_only ? 6 : (7 + L);
#define SOLVE_EV(k) do { if (MEGA && tid == 0) log_event(log, ev_desc(EV_SOLVE_PHASE, 0, o, k)); } while (0)
  SOLVE_EV(0);
  const bool dbg = (a.dbg_H != nullptr);
  const bool use_render = !pose_only && !prm.sdf_only;
  // tile partials of this object, summed in tile order (deterministic), fp64
  const int V = ldv(b.V_count + o), m = use_render ? ldv(b.band_m + o) : 0;
  const int ntS = (b.meta[o].n_pts + a.tile_rows - 1) / a.tile_rows;
  const int ntR = use_render ? (m + a.tile_rows - 1) / a.tile_rows : 0;
  const float* pS = a.part_s + (size_t)a.base_s[o] * kAccStride;
  const float* pR = use_render ? a.part_r + (size_t)a.base_r[o] * kAccStride : nullptr;
  // ---- losses and the reference's soft-failure exits (optimizer.py:130-150) -----------------
  if (ldv(&st.status) != 0) {                    // frozen object: keep its record
    if (last_iter && tid == 0 && !dbg) write_result(b, o, st);
    return 1;
  }
  if (tid < 96) {
    // three fixed-order reductions over the tiles (lane-strided partial sums + xor butterfly): warp 0: SDF
    // loss, warp 1: SDF row count, warp 2: render loss
    const int w = tid >> 5, ln = tid & 31;
    const float* src = (w < 2) ? pS : pR;
    const int nt = (w < 2) ? ntS : ntR, idx = (w == 1) ? kAccLoss + 1 : kAccLoss;
    double v = 0.0;
    for (int t = ln; t < nt; t += 32) v += (double)__ldcg(src + (size_t)t * kAccStride + idx);
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) v += __shfl_xor_sync(0xffffffffu, v, d);
    if (ln == 0) s_sum[w] = v;
  }
  solve_sync<MEGA>();
  SOLVE_EV(1);
  const double nS = s_sum[1];
  const float sdf_loss = (float)(s_sum[0] / nS);
  float render_loss = 0.f;
  int status = 0;
  if (isnan(sdf_loss)) status = DSPGN_ST_SDF_NAN;
  else if (use_render) {
    if (V < 10) status = DSPGN_ST_RENDER_FEW;
    else {
      render_loss = (m > 0) ? (float)(s_sum[2] / (double)m) : NAN;
      if (isnan(render_loss)) status = DSPGN_ST_RENDER_NAN;
    }
  }
  if (dbg && o == a.dbg_obj && tid == 0) {
    a.dbg_loss[0] = sdf_loss; a.dbg_loss[1] = render_loss; a.dbg_loss[2] = (float)V; a.dbg_loss[3] = (float)m;
  }
  if (status != 0) {
    if (!dbg && tid == 0) { st.status = status; st.V = V; st.m = m; if (last_iter || MEGA) write_result(b, o, st); }
    return 1;
  }
  // optimizer.py:155.  The contraction is spelled out: left to the compiler, which product it fuses depends on the
  // surrounding code, and both schedules (k_solve, the persistent kernel) must round alike.
  const float loss = __fmaf_rn(prm.k1, render_loss, __fmul_rn(prm.k2, sdf_loss));

  if (tid == 0) {
    s_flag = 0;
    s_rot[0] = s_rot[1] = s_rot[2] = s_rot[3] = 0.f;
    if (!pose_only) {
      // rotation prior (loss.py:155-178): r = 1 - (R_co e_y).n_g, n_g = (0,-1,0)
      float Toc[12], Tco[12];
      double det_oc;
      for (int i = 0; i < 12; ++i) Toc[i] = ldv(&st.T_oc[i]);
      inv_affine(Toc, Tco, &det_oc);
      const float scale = powf((float)(1.0 / det_oc), 1.0f / 3.0f);
      float rco[12];
      for (int i = 0; i < 12; ++i) rco[i] = Tco[i] / scale;
      rco[3] = rco[7] = rco[11] = 0.f;
      float roc[12];
      inv_affine(rco, roc, nullptr);
      const float res_rot = 1.0f + rco[1 * 4 + 1];                     // 1 - dot(R_co[:,1], (0,-1,0))
      if (!(res_rot < 1e-7f)) {
        // v = R_oc n_g = -R_oc[:,1];  J_rot = v x e_y = (-v_z, 0, v_x)
        s_rot[0] = roc[2 * 4 + 1];      // -v_z
        s_rot[1] = -roc[0 * 4 + 1];     //  v_x
        s_rot[2] = res_rot;
        s_rot[3] = 1.f;
      }
    }
  }
  solve_sync<MEGA>();

  SOLVE_EV(2);
  // ---- assemble the lower triangle of H and the b row (optimizer.py:161-184; pose-only: :68-71) ----
  const double wS = pose_only ? 1.0 / nS : (double)prm.k2 / nS;
  const double wR = use_render ? (double)prm.k1 / (double)m : 0.0;
  // Entry e = tid + q*256 of a tile partial: e < kTriInt -> packed upper-triangle element (r, c) of the internal matrix,
  // then the 72 b entries.  Consecutive threads read consecutive floats.  (i, j) = position in the EXTERNAL system
  // [pose | code] with i >= j, i == P for a right-hand-side entry, i = -1 for an entry that is not part of this system
  // (padding column 71, code rows >= code_len, every code row in a pose-only run).
  auto int_to_ext = [&](int r) -> int {
    if (r >= kMaxCode) { const int p = r - kMaxCode; return (p < npose) ? p : -1; }
    return (!pose_only && r < L) ? npose + r : -1;
  };
  int ei[kMaxEnt], ej[kMaxEnt], eidx[kMaxEnt];
  double accv[kMaxEnt], accr[kMaxEnt];
#pragma unroll
  for (int q = 0; q < kMaxEnt; ++q) {
    const int e = tid + q * kSolveThreads;
    int i = -1, j = 0, idx = 0;
    if (e < kTriInt) {
      // invert tri_index: base(r) = r (145 - r) / 2 <= e
      int r = (int)((145.f - sqrtf(21025.f - 8.f * (float)e)) * 0.5f);
      r = max(0, min(r, kPInt - 1));
      while (r + 1 < kPInt && tri_index(r + 1, r + 1) <= e) ++r;
      while (tri_index(r, r) > e) --r;
      const int c = r + (e - tri_index(r, r));
      const int xi = int_to_ext(r), xj = int_to_ext(c);
      if (xi >= 0 && xj >= 0) { i = max(xi, xj); j = min(xi, xj); }
      idx = e;
    } else if (e < kTriInt + kPInt) {
      const int xj = int_to_ext(e - kTriInt);
      if (xj >= 0) { i = P; j = xj; }
      idx = kAccB + (e - kTriInt);
    }
    ei[q] = i; ej[q] = j; eidx[q] = idx;
    accv[q] = 0.0; accr[q] = 0.0;
  }
  // tile partials summed in tile order; the thread's (up to 11) entries give 11 independent loads per tile
  // (four tiles' loads are issued before their sums: 44 independent L2 round trips in flight per thread; the
  //  summation order -- tile 0, 1, 2, ... -- is unchanged)
  auto sum_tiles = [&](const float* base, int nt, double (&acc)[kMaxEnt]) {
    int t = 0;
    for (; t + 4 <= nt; t += 4) {
      float v[4][kMaxEnt];
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const float* pt = base + (size_t)(t + u) * kAccStride;
#pragma unroll
        for (int q = 0; q < kMaxEnt; ++q) v[u][q] = (ei[q] >= 0) ? __ldcg(pt + eidx[q]) : 0.f;
      }
#pragma unroll
      for (int u = 0; u < 4; ++u)
#pragma unroll
        for (int q = 0; q < kMaxEnt; ++q) acc[q] += (double)v[u][q];
    }
    for (; t < nt; ++t) {
      const float* pt = base + (size_t)t * kAccStride;
#pragma unroll
      for (int q = 0; q < kMaxEnt; ++q) if (ei[q] >= 0) acc[q] += (double)__ldcg(pt + eidx[q]);
    }
  };
  sum_tiles(pS, ntS, accv);
  if (ntR > 0) sum_tiles(pR, ntR, accr);
  SOLVE_EV(3);
#pragma unroll
  for (int q = 0; q < kMaxEnt; ++q) {
    const int i = ei[q], j = ej[q];
    if (i < 0) continue;
    double v;
    if (i < P) {
      v = wS * accv[q] + wR * accr[q];
      if (pose_only) {
        if (i == j) v += 1e-2;                                           // optimizer.py:70
      } else {
        if (i == j && i >= 7) v += (double)prm.k3;                       // optimizer.py:170
        if (i == j && i < 7) v += 1.0;                                   // optimizer.py:182
        if (i == 6 && j == 6) v += (double)prm.s_damp;                   // optimizer.py:183
        if (s_rot[3] != 0.f && i >= 3 && i < 6 && j >= 3) {              // optimizer.py:176-178
          const double Ji = (i == 3) ? s_rot[0] : (i == 5 ? s_rot[1] : 0.0);
          const double Jj = (j == 3) ? s_rot[0] : (j == 5 ? s_rot[1] : 0.0);
          v += (double)prm.k4 * Ji * Jj;
        }
      }
      if (dbg && o == a.dbg_obj) { a.dbg_H[i * P + j] = (float)v; a.dbg_H[j * P + i] = (float)v; }
    } else {
      v = -(wS * accv[q] + wR * accr[q]);
      if (!pose_only) {
        if (j >= 7) v -= (double)prm.k3 * (double)ldv(&st.z[j - 7]);     // optimizer.py:172
        if (s_rot[3] != 0.f && (j == 3 || j == 5))                       // optimizer.py:177-179 sign
          v += (double)prm.k4 * (double)(j == 3 ? s_rot[0] : s_rot[1]) * (double)s_rot[2];
      }
      if (dbg && o == a.dbg_obj) a.dbg_b[j] = (float)v;
    }
    if (i < P) { As[i * kAsStride + j] = (float)v; As[j * kAsStride + i] = (float)v; }
    else As[j * kAsStride + kPMax] = (float)v;           // b_j -> augmented column
  }
  solve_sync<MEGA>();
  // this iteration's H without the damping overwrites the slot's last linearisation (every successful assembly, so the
  // buffer holds the system of the iteration the record's final update came from).  A pass of its own over the
  // assembled rows, warp per row: written inside the assembly loop above, the store measured slower on every run,
  // including the runs that keep nothing.  The damping comes off the fp32 entry in fp64: at most half an ulp of the
  // damped entry (with scale_damping 100, 4e-6 on the scale diagonal).
  if (b.lin != nullptr && !dbg) {
    float* lin = b.lin + (size_t)o * lin_floats(L);
    const int lane = tid & 31;
    for (int r = tid >> 5; r < P; r += kSolveThreads / 32) {
      float* row = lin + lin_index(r, r, P) - r;
      for (int c = r + lane; c < P; c += 32) {
        const double damp = pose_only ? (r == c ? 1e-2 : 0.0)
                                      : (r == c && r < 7 ? (r == 6 ? 1.0 + (double)prm.s_damp : 1.0) : 0.0);
        row[c] = (float)((double)As[r * kAsStride + c] - damp);
      }
    }
  }

  // padding rows/columns P..70 (pose-only: P = 6): identity, zero right-hand side
  for (int idx = tid; idx < kPMax * (kPMax + 1); idx += kSolveThreads) {
    const int i = idx / (kPMax + 1), j = idx - i * (kPMax + 1);
    if (i >= P || (j >= P && j < kPMax)) As[i * kAsStride + j] = (i == j) ? 1.f : 0.f;
  }
  solve_sync<MEGA>();
  SOLVE_EV(4);
  // the stop word: read by the first thread the elimination leaves idle, so its PCIe round trip runs under the pivots
  // (the barrier after the elimination publishes it; a failed solve ignores it)
  if (tid == kElimThreads && !dbg) SM.s_stop = stop_check(b.stop, o, ldv(&st.iters), pose_only, last_iter);
  // ---- Gauss-Jordan elimination of the SPD system, thread i = row i in registers; one barrier per pivot ----------
  if (tid < kElimThreads) {
    // Thread i keeps row i of [H | b] in registers, rotated so that the current pivot column is always index 0: after
    // pivot k, arow[j] holds H'[i][k+1+j].  The pivot loop stays rolled (small, cache-resident code) while every register
    // index is a compile-time constant.  Rows ABOVE the pivot are eliminated too (Jordan), so the system ends diagonal
    // and x_i = b'_i / H'_ii with the diagonal each thread saved when its own row was the pivot: no U factor in shared
    // memory and no back-substitution chain (71 more dependent barrier steps in the previous version).
    float arow[kPMax + 1];
    const int row = (tid < kPMax) ? tid : kPMax - 1;        // lanes 71..95 mirror the last row (results unused)
#pragma unroll
    for (int j = 0; j < kPMax; ++j) arow[j] = As[row * kAsStride + j];
    arow[kPMax] = 0.f;
    float brow = As[row * kAsStride + kPMax];
    float mydiag = 1.f;
    int bad_pivot = 0;
    // After k rotations only entries 0 .. 70-k of a rotated row can be non-zero, so the pivots run in three tiers that
    // broadcast / load / update only the first 72, 48 and 24 entries (whole loop bodies specialised at compile time --
    // per-chunk branches inside one body measured slower than no skipping at all).
    gj_pivots<18>(0, 24, tid, arow, brow, mydiag, bad_pivot, bcast);
    gj_pivots<12>(24, 48, tid, arow, brow, mydiag, bad_pivot, bcast);
    gj_pivots<6>(48, kPMax, tid, arow, brow, mydiag, bad_pivot, bcast);
    if (tid < kPMax) xs[tid] = brow / mydiag;
    if (bad_pivot && tid == 0) s_flag = 1;
  }
  solve_sync<MEGA>();
  SOLVE_EV(5);
  if (tid < P && !isfinite(xs[tid])) s_flag = 1;
  solve_sync<MEGA>();
  if (dbg) {
    if (o == a.dbg_obj && tid < P) a.dbg_dx[tid] = xs[tid];
    return 1;
  }
  // ---- update (optimizer.py:186-192 / :72-74), clear accumulators, next depth range -----------
  const bool fail = (s_flag != 0);
  if (!pose_only && tid < L && !fail) st.z[tid] = ldv(&st.z[tid]) + prm.lr * xs[tid + 7];
  solve_sync<MEGA>();                        // the result record below reads every z entry
  // a stop observed in this solve ends the object as its last iteration would: the same update, the same record but
  // the status
  const bool stop = !fail && SM.s_stop != 0;
  const bool final_solve = last_iter || stop;
  if (!pose_only && !fail && !final_solve) refresh_zb0(st, b.decs[b.meta[o].class_id], tid, kSolveThreads);
  if (tid == 0) {
    st.loss = loss; st.V = V; st.m = m;
    b.V_count[o] = 0;
    if (fail) {
      st.status = DSPGN_ST_SOLVE;
    } else {
      float dp[7];
      for (int i = 0; i < npose; ++i) dp[i] = (pose_only ? 1.0f : prm.lr) * xs[i];
      float dT[12], Tn[12], Toc[12];
      for (int i = 0; i < 12; ++i) Toc[i] = ldv(&st.T_oc[i]);
      exp_sim3_dev(dp, !pose_only, dT);
      mul_affine(dT, Toc, Tn);
      for (int i = 0; i < 12; ++i) st.T_oc[i] = Tn[i];
      derive_depth_range(st, prm.D);
      st.iters = ldv(&st.iters) + 1;
    }
    if (stop) { st.status = DSPGN_ST_STOPPED; st.n_iter = st.iters; }   // later launches skip it (k_solve, term_rows)
    if (final_solve || (MEGA && fail)) write_result(b, o, st);
  }
  SOLVE_EV(6);
  return (final_solve || fail) ? 1 : 0;
}

__global__ void __launch_bounds__(kSolveThreads) k_solve(BatchDev b, SolveArgs a) {
  __shared__ SolveSmem SM;
  const int o = blockIdx.x, n_iter = b.state[o].n_iter;
  if (a.iter_index >= n_iter) return;               // finished after its own last iteration
  const bool last = a.iter_index + 1 == n_iter;
  solve_object<false>(b, a, EventLog{}, o, threadIdx.x, SM, last);
  // gated pose-only object: the map-consistency check on the record thread 0 has just written
  if (last && b.link != nullptr && a.dbg_H == nullptr && threadIdx.x == 0 && b.link[o] >= 0 && b.state[o].mode == DSPGN_MODE_POSE)
    gate_record(b.results, o, b.T_init, b.t_map);
}

// Per-iteration schedule of a gated run, between its two phases: the joint slots whose pose-only object was rejected
// run num_iterations from their k_init state, every other object is finished (its record is final).  Once the call's
// stop is observed no slot wakes: a rejected one gets its stopped record.
__global__ void k_gate_wake(BatchDev b, int n_iter_joint) {
  const int o = blockIdx.x * blockDim.x + threadIdx.x;
  if (o >= b.n_obj) return;
  const int lk = b.link[o];
  bool wake = lk >= 0 && b.modes[o] == DSPGN_MODE_JOINT &&
              reinterpret_cast<const int*>(b.results + (size_t)lk * DSPGN_RESULT_FLOATS)[85] == DSPGN_GATE_REJECTED;
  if (wake && b.stop.word != nullptr && stop_seen(b.stop)) {
    stopped_slot_record(b.results, b.state, b.T_init, o);
    wake = false;
  }
  b.state[o].n_iter = wake ? n_iter_joint : 0;
}

// dspgn_keyframe_batch_meshed, after the run's last iteration (both schedules): which objects get a mesh.  One CTA per
// object.  grid_slot[o] >= 0 marks a candidate (a joint object, including the joint slot of a gated object); pair[o] is the
// other hypothesis of a mono pair (-1: none).  Writes the record's mesh word, and for a DSPGN_MESH_DONE object the layer-0
// bias folded from its final code (the solve does not refresh zb0 after the last iteration) for the MODE_GRIDFWD decode.
__global__ void k_mesh_select(BatchDev b, const int* grid_slot, const int* pair) {
  const int o = blockIdx.x, tid = threadIdx.x;
  __shared__ int s_word;
  if (tid == 0) {
    const int* rec = reinterpret_cast<const int*>(b.results);
    const float* recf = b.results;
    const size_t RF = DSPGN_RESULT_FLOATS;
    int word = DSPGN_MESH_OFF;
    const int lk = (b.link != nullptr) ? b.link[o] : -1;
    // the joint slot of a gated object is a candidate only when the device rejected its pose-only record
    const bool woken = lk < 0 || rec[(size_t)lk * RF + 85] == DSPGN_GATE_REJECTED;
    if (grid_slot[o] >= 0 && woken) {
      const int p = pair[o];
      // the pair rule of ProcessDetectedObjects (src/LocalMapping_util.cc:403-407): hypothesis j > i wins iff
      // loss[i] > loss[j]; a tie keeps i
      const bool lost = p >= 0 && (p > o ? recf[(size_t)o * RF + 80] > recf[(size_t)p * RF + 80]
                                         : !(recf[(size_t)p * RF + 80] > recf[(size_t)o * RF + 80]));
      word = lost ? DSPGN_MESH_LOST : (rec[(size_t)o * RF + 81] != DSPGN_ST_OK ? DSPGN_MESH_FAILED : DSPGN_MESH_DONE);
    }
    reinterpret_cast<int*>(b.results + (size_t)o * RF)[kRecMeshWord] = word;
    s_word = word;
  }
  __syncthreads();
  if (s_word == DSPGN_MESH_DONE) refresh_zb0(b.state[o], b.decs[b.meta[o].class_id], tid, blockDim.x);
}

// ---- pose information of a record (dspgn_pose_information, DESIGN §4.13) -------------------------------------------
// One per object of the call: the BatchDev::lin slot its record came from (-1: no valid linearisation), that slot's P (6
// pose-only, 7 + L joint) and the scale s of the map into the object edge's tangent space.
struct InfoItem { int slot; int P; double s; };
constexpr int kInfoThreads = 128;

// One CTA per object, fp64.  The Schur complement of the slot's H onto the six pose coordinates (scale and code
// eliminated, last index first), a Cholesky test of that 6x6 block, then the map from the library's left perturbation
// delta = [rho | phi] of T_obj_cam to the edge's e = [omega | upsilon] (Z exp(e)): delta = (-upsilon / s, -omega), so
// Lambda[a][b] = f_a f_b M[p_a][p_b] with p = (3, 4, 5, 0, 1, 2), f = (-1, -1, -1, -1/s, -1/s, -1/s).
__global__ void __launch_bounds__(kInfoThreads) k_pose_information(const float* lin, int stride, const InfoItem* items,
                                                                   double* info, int* status) {
  __shared__ double A[kPMax][kPMax + 1];       // lower triangle (i >= j) of the system being reduced
  __shared__ int s_ok;
  const int o = blockIdx.x, tid = threadIdx.x;
  const InfoItem it = items[o];
  double* out = info + 36 * (size_t)o;
  const int P = it.P;
  if (tid == 0) s_ok = it.slot >= 0 && (P == 6 || (P > 7 && P <= kPMax)) && it.s > 0.0 && isfinite(it.s);
  __syncthreads();
  if (s_ok) {
    const float* h = lin + (size_t)it.slot * stride;
    for (int e = tid; e < P * P; e += kInfoThreads) {
      const int i = e / P, j = e - i * P;
      if (j <= i) A[i][j] = (double)h[lin_index(j, i, P)];
    }
    __syncthreads();
    for (int k = P - 1; k >= 6; --k) {
      const double d = A[k][k];                  // the same shared value in every thread: a uniform exit
      if (!(d > 0.0) || !isfinite(d)) { if (tid == 0) s_ok = 0; break; }
      for (int e = tid; e < k * k; e += kInfoThreads) {
        const int i = e / k, j = e - i * k;
        if (j <= i) A[i][j] -= A[k][i] * A[k][j] / d;
      }
      __syncthreads();
    }
    __syncthreads();
    if (tid == 0 && s_ok) {                      // positive definite: Cholesky of the marginal 6x6 block
      double Lc[6][6];
      for (int i = 0; i < 6 && s_ok; ++i)
        for (int j = 0; j <= i; ++j) {
          double v = A[i][j];
          for (int q = 0; q < j; ++q) v -= Lc[i][q] * Lc[j][q];
          if (i == j) {
            if (!(v > 0.0) || !isfinite(v)) { s_ok = 0; break; }
            Lc[i][i] = sqrt(v);
          } else {
            Lc[i][j] = v / Lc[j][j];
          }
        }
    }
    __syncthreads();
  }
  if (tid < 36) {
    const int a = tid / 6, c = tid - a * 6;
    double v = 0.0;
    if (s_ok) {
      const int pa = a < 3 ? a + 3 : a - 3, pc = c < 3 ? c + 3 : c - 3;
      const double fa = a < 3 ? -1.0 : -1.0 / it.s, fc = c < 3 ? -1.0 : -1.0 / it.s;
      v = fa * fc * A[max(pa, pc)][min(pa, pc)];
    }
    out[tid] = v;
  }
  if (tid == 0) status[o] = s_ok ? DSPGN_INFO_OK : DSPGN_INFO_NONE;
}

// ---------------------------------------------------------------------------------------------
// Render term, per-ray part (loss.py:84-141).  One CTA per object, one warp per ray, two passes:
// pass 1 counts the band samples each ray keeps, a block scan turns counts into row offsets, pass 2
// recomputes and writes rows (x_o, de/ds, clamped depth residual) in (ray, sample) order -- the same
// order torch.where yields, and deterministic.  th: the occupancy cut-off (SolverParams::th).
constexpr int kScanThreads = 1024;
constexpr int kScanMaxRays = 8192;
static_assert((long long)kScanMaxRays * kMaxDepthSamples <= (1LL << (31 - kRangeSampleBits)),
              "an object's sample count must fit the range word's prefix field");

// pose / depth range of the object being scanned, read once per thread (cache-bypassing: in the persistent kernel
// another CTA's solve wrote it)
struct ScanState { float T[12]; float dmin, dmax, dstep, dfar; };
__device__ __forceinline__ void load_scan_state(const ObjState& st, ScanState& c) {
#pragma unroll
  for (int i = 0; i < 12; ++i) c.T[i] = ldv(&st.T_oc[i]);
  c.dmin = ldv(&st.dmin); c.dmax = ldv(&st.dmax); c.dstep = ldv(&st.dstep); c.dfar = ldv(&st.dfar);
}

// sdf values of one ray (lane = sample slot, two slots per lane); +inf beyond D / outside the unit sphere
__device__ __forceinline__ void ray_load(const BatchDev& b, const ObjMeta& M, int ray, int lane, float s[2]) {
  const float* srow = b.sdf + (size_t)M.smp_off + (size_t)ray * b.D;
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int j = lane + 32 * h;
    s[h] = (j < b.D) ? __ldcg(srow + j) : INFINITY;  // written by other CTAs (L2 is the point of coherence)
  }
}

// same for the compact layout: the ray's hull [j0, j0 + cnt) starts at sample slot `p` of the object
__device__ __forceinline__ void ray_load_compact(const BatchDev& b, const ObjMeta& M, int p, int j0, int cnt, int lane, float s[2]) {
  const float* srow = b.sdf + (size_t)M.smp_off + (size_t)p;
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int k = lane + 32 * h - j0;
    s[h] = (k >= 0 && k < cnt) ? __ldcg(srow + k) : INFINITY;
  }
}

__device__ __forceinline__ void ray_scan_vals(const BatchDev& b, const float th, const ObjMeta& M, const ScanState& st, int ray,
                                              int lane, const float s[2], bool keep[2], float de_ds[2], float& res) {
  const int D = b.D;
  float o[2], q[2];
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int j = lane + 32 * h;
    o[h] = (j < D) ? occupancy(s[h], th) : 0.f;      // +inf -> clamp -> 0 (outside sphere: loss.py:84)
    q[h] = 1.f - o[h];
  }
  // inclusive product scan over the 64 slots -> transmittance T_l (loss.py:99)
  float t0 = q[0], t1 = q[1];
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    float y0 = __shfl_up_sync(0xffffffffu, t0, d), y1 = __shfl_up_sync(0xffffffffu, t1, d);
    if (lane >= d) { t0 *= y0; t1 *= y1; }
  }
  const float tot0 = __shfl_sync(0xffffffffu, t0, 31);
  t1 *= tot0;
  float T[2] = {t0, t1};
  // termination probabilities and rendered depth (loss.py:100-114)
  float Tprev0 = __shfl_up_sync(0xffffffffu, t0, 1);
  float Tprev1 = __shfl_up_sync(0xffffffffu, t1, 1);
  if (lane == 0) { Tprev0 = 1.f; Tprev1 = tot0; }
  float du = 0.f;
  if (lane < D) du += lin_depth(st.dmin, st.dmax, st.dstep, lane, D) * (o[0] * Tprev0);
  if (lane + 32 < D) du += lin_depth(st.dmin, st.dmax, st.dstep, lane + 32, D) * (o[1] * Tprev1);
  const int jl = D - 1;                                   // T_{D-1}
  const float Tlast = __shfl_sync(0xffffffffu, (jl >= 32) ? T[1] : T[0], jl & 31);
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) du += __shfl_xor_sync(0xffffffffu, du, d);
  du += st.dfar * Tlast;
  // suffix sums S_j = sum_{l >= j} T_l (loss.py:118-122); slots >= D contribute 0
  float u0 = (lane < D) ? T[0] : 0.f, u1 = (lane + 32 < D) ? T[1] : 0.f;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    float y0 = __shfl_down_sync(0xffffffffu, u0, d), y1 = __shfl_down_sync(0xffffffffu, u1, d);
    if (lane + d < 32) { u0 += y0; u1 += y1; }
  }
  const float hi_tot = __shfl_sync(0xffffffffu, u1, 0);
  u0 += hi_tot;
  const float S[2] = {u0, u1};
  const float delta_d = (st.dmax - st.dmin) / (float)(D - 1);
  const float do_ds = -1.0f / (2.0f * th);
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const bool band = (s[h] > -th) && (s[h] < th);      // loss.py:88 (strict); inf never passes
    const float de_do = S[h] / (1.f - o[h]);
    keep[h] = band && (de_do > 1e-2f);                  // loss.py:125
    de_ds[h] = de_do * delta_d * do_ds;                 // loss.py:128-130
  }
  const float dobs = (ray < M.n_fg) ? b.depth_fg[M.fg_off + ray] : st.dfar;   // optimizer.py:126
  res = fminf(fmaxf(dobs - du, -0.3f), 0.3f);           // loss.py:136-141
}

__device__ __forceinline__ void ray_scan(const BatchDev& b, const float th, const ObjMeta& M, const ScanState& st, int ray, int lane,
                                         bool keep[2], float de_ds[2], float& res) {
  float s[2];
  ray_load(b, M, ray, lane, s);
  ray_scan_vals(b, th, M, st, ray, lane, s, keep, de_ds, res);
}

// write the kept samples of one ray as band rows (x_o, de/ds, residual) starting at row `base` (ray, sample order);
// the two slots hold samples j0 + lane and j0 + lane + 32
__device__ __forceinline__ int ray_emit(const BatchDev& b, const ObjMeta& M, const ScanState& st, int ray, int lane,
                                        const bool keep[2], const float de_ds[2], float res, size_t base, int j0 = 0) {
  const unsigned b0 = __ballot_sync(0xffffffffu, keep[0]), b1 = __ballot_sync(0xffffffffu, keep[1]);
  const float* q = b.rays + 3 * (size_t)(M.ray_off + ray);
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    if (!keep[h]) continue;
    const int j = j0 + lane + 32 * h;
    const int pos = (h == 0 ? __popc(b0 & ((1u << lane) - 1u)) : __popc(b0) + __popc(b1 & ((1u << lane) - 1u)));
    const float d = lin_depth(st.dmin, st.dmax, st.dstep, j, b.D);
    float x, y, z;
    xform_point(st.T, __fmul_rn(q[0], d), __fmul_rn(q[1], d), __fmul_rn(q[2], d), x, y, z);
    const size_t row = base + pos;
    b.band_x[3 * row] = x; b.band_x[3 * row + 1] = y; b.band_x[3 * row + 2] = z;
    b.band_s[row] = de_ds[h];
    b.band_r[row] = res;
  }
  return __popc(b0) + __popc(b1);
}

// ---- long rays (D > 64): the same render term, walked in windows of 64 samples -------------------------------------
// Window w holds samples 64w + lane + 32h in ray_scan_vals' two-slot lane layout; D is the same for every ray of a call,
// so the choice between the two paths is warp-uniform.  Two passes over the windows, each reloading the window's sdf
// values from L2 (no register array grows with D):
//   forward: the running transmittance Tc (product of 1 - o over the earlier windows; loss.py:99), each lane's part of
//            the rendered depth (loss.py:100-114), T at the last sample and the finite-value count; lane w keeps window
//            w's Tc and its sum of T.  The suffix sum after each window (sum of T over the later windows) is then carried
//            backwards across those lane words (loss.py:118-122).
//   emit:    each window's scan again from its Tc, its suffix sums from that carry, then the band test, de/ds and the
//            rows (loss.py:125-141) at the ray's running row count, so rows stay in (ray, sample) order.
constexpr int kLongWin = 64, kLongMaxWin = kMaxDepthSamples / kLongWin;
static_assert(kLongMaxWin <= 32, "one lane word per window");

// one window: occupancies, T = Tc x the inclusive product scan of 1 - o, and the window's suffix sums of T (samples < D)
__device__ __forceinline__ void long_window(const float th, int D, int j0, int lane, float Tc, const float s[2], float o[2],
                                            float T[2], float S[2]) {
  float t[2];
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    o[h] = (j0 + lane + 32 * h < D) ? occupancy(s[h], th) : 0.f;
    t[h] = 1.f - o[h];
  }
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const float y0 = __shfl_up_sync(0xffffffffu, t[0], d), y1 = __shfl_up_sync(0xffffffffu, t[1], d);
    if (lane >= d) { t[0] *= y0; t[1] *= y1; }
  }
  t[1] *= __shfl_sync(0xffffffffu, t[0], 31);
  T[0] = Tc * t[0]; T[1] = Tc * t[1];
  float u0 = (j0 + lane < D) ? T[0] : 0.f, u1 = (j0 + lane + 32 < D) ? T[1] : 0.f;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const float y0 = __shfl_down_sync(0xffffffffu, u0, d), y1 = __shfl_down_sync(0xffffffffu, u1, d);
    if (lane + d < 32) { u0 += y0; u1 += y1; }
  }
  S[0] = u0 + __shfl_sync(0xffffffffu, u1, 0); S[1] = u1;
}

// One long ray: its sdf values are samples [first, first + cnt) at b.sdf + M.smp_off + p (the n_rays x D layout is
// p = ray * D, first = 0, cnt = D).  Adds the ray's finite values to nvalid; with `emit`, writes its kept samples as band
// rows from row `base`.  Returns the kept count.  All 32 lanes.
__device__ inline int long_ray(const BatchDev& b, const float th, const ObjMeta& M, const ScanState& st, int ray, int lane,
                               int p, int first, int cnt, bool emit, size_t base, int& nvalid) {
  const int D = b.D, nwin = (D + kLongWin - 1) / kLongWin;
  float s[2], o[2], T[2], S[2];
  float Tc = 1.f, du = 0.f, Tlast = 0.f, wTc = 0.f, wsum = 0.f;   // wTc / wsum: lane w holds window w's
#pragma unroll 1
  for (int w = 0; w < nwin; ++w) {
    const int j0 = w * kLongWin;
    ray_load_compact(b, M, p, first - j0, cnt, lane, s);
    nvalid += __popc(__ballot_sync(0xffffffffu, s[0] != INFINITY)) + __popc(__ballot_sync(0xffffffffu, s[1] != INFINITY));
    long_window(th, D, j0, lane, Tc, s, o, T, S);
    float Tprev0 = __shfl_up_sync(0xffffffffu, T[0], 1), Tprev1 = __shfl_up_sync(0xffffffffu, T[1], 1);
    const float mid = __shfl_sync(0xffffffffu, T[0], 31);
    if (lane == 0) { Tprev0 = Tc; Tprev1 = mid; }
    if (j0 + lane < D) du += lin_depth(st.dmin, st.dmax, st.dstep, j0 + lane, D) * (o[0] * Tprev0);
    if (j0 + lane + 32 < D) du += lin_depth(st.dmin, st.dmax, st.dstep, j0 + lane + 32, D) * (o[1] * Tprev1);
    const int jl = D - 1 - j0;                                // T_{D-1}, in the last window
    if (jl < kLongWin) Tlast = __shfl_sync(0xffffffffu, (jl >= 32) ? T[1] : T[0], jl & 31);
    const float sum = __shfl_sync(0xffffffffu, S[0], 0);
    if (lane == w) { wTc = Tc; wsum = sum; }
    Tc = __shfl_sync(0xffffffffu, T[1], 31);
  }
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) du += __shfl_xor_sync(0xffffffffu, du, d);
  du += st.dfar * Tlast;
  const float dobs = (ray < M.n_fg) ? b.depth_fg[M.fg_off + ray] : st.dfar;   // optimizer.py:126
  const float res = fminf(fmaxf(dobs - du, -0.3f), 0.3f);                    // loss.py:136-141
  float wsuf = 0.f, carry = 0.f;                            // lane w: sum of T over the windows after w
#pragma unroll 1
  for (int w = nwin - 1; w >= 0; --w) {
    if (lane == w) wsuf = carry;
    carry += __shfl_sync(0xffffffffu, wsum, w);
  }
  const float delta_d = (st.dmax - st.dmin) / (float)(D - 1);
  const float do_ds = -1.0f / (2.0f * th);
  int count = 0;
#pragma unroll 1
  for (int w = 0; w < nwin; ++w) {
    const int j0 = w * kLongWin;
    ray_load_compact(b, M, p, first - j0, cnt, lane, s);
    long_window(th, D, j0, lane, __shfl_sync(0xffffffffu, wTc, w), s, o, T, S);
    const float after = __shfl_sync(0xffffffffu, wsuf, w);
    bool keep[2]; float de_ds[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const bool band = (s[h] > -th) && (s[h] < th);    // loss.py:88 (strict); inf never passes
      const float de_do = (S[h] + after) / (1.f - o[h]);
      keep[h] = band && (de_do > 1e-2f);                // loss.py:125
      de_ds[h] = de_do * delta_d * do_ds;               // loss.py:128-130
    }
    if (emit) count += ray_emit(b, M, st, ray, lane, keep, de_ds, res, base + count, j0);
    else count += __popc(__ballot_sync(0xffffffffu, keep[0])) + __popc(__ballot_sync(0xffffffffu, keep[1]));
  }
  return count;
}

// ---- persistent kernel: the scan as parallel work items --------------------------------------------------------------
// A scan item covers kScanChunkRays consecutive rays of one object; warp w of the CTA's 8 epilogue warps owns the
// "segment" of kSegRays rays  [chunk*64 + 8w, +8)  and writes its kept rows compactly at the START of the segment's own
// sample range (single pass, all sdf loads of the segment issued up front).  Band rows keep the global (ray, sample)
// order; band tiles find them through the per-object exclusive prefix over the segment counts.
constexpr int kSegRays = 8, kScanChunkRays = 64;
// first segment slot of object o: its nseg counts / nseg + 1 prefix entries never overlap the next object's
__device__ __forceinline__ int seg_base(const ObjMeta& M, int o) { return M.ray_off / kSegRays + 2 * o; }

// vpre: the compact sdf layout of valid_sample_ranges, nullptr = n_rays x D
__device__ inline void scan_chunk(const BatchDev& b, const float th, const int* vpre, int* seg_cnt, const int o, const int chunk,
                                  const int tid) {
  const int lane = tid & 31, warp = tid >> 5;
  const ObjMeta M = b.meta[o];
  const int seg = chunk * (kScanChunkRays / kSegRays) + warp;
  const int ray0 = seg * kSegRays;
  if (ray0 >= M.n_rays) return;
  ScanState st;
  load_scan_state(b.state[o], st);
  // compact sdf layout: lanes 0..8 fetch the segment's 9 range words once
  int vw = 0;
  if (vpre != nullptr && lane <= kSegRays && ray0 + lane <= M.n_rays) vw = __ldcg(vpre + vpre_base(M, o) + ray0 + lane);
  const size_t base = (size_t)M.smp_off + (size_t)ray0 * b.D;
  if (b.D > kLongWin) {                                    // long rays: one ray at a time, rows at the segment's head
    int nvalid = 0, count = 0;
#pragma unroll 1
    for (int i = 0; i < kSegRays; ++i) {
      const int v0 = __shfl_sync(0xffffffffu, vw, i), v1 = __shfl_sync(0xffffffffu, vw, i + 1);
      const int ray = ray0 + i;
      if (ray >= M.n_rays) break;                          // warp-uniform
      const int p = vpre != nullptr ? v0 >> kRangeSampleBits : ray * b.D;
      const int first = vpre != nullptr ? v0 & kRangeSampleMask : 0;
      const int cnt = vpre != nullptr ? (v1 >> kRangeSampleBits) - (v0 >> kRangeSampleBits) : b.D;
      count += long_ray(b, th, M, st, ray, lane, p, first, cnt, true, base + count, nvalid);
    }
    if (lane == 0 && nvalid != 0) atomicAdd(b.V_count + o, nvalid);
    if (lane == 0) seg_cnt[seg_base(M, o) + seg] = count;
    return;
  }
  float sv[kSegRays][2];
#pragma unroll
  for (int i = 0; i < kSegRays; ++i) {
    const int v0 = __shfl_sync(0xffffffffu, vw, i), v1 = __shfl_sync(0xffffffffu, vw, i + 1);
    if (ray0 + i < M.n_rays) {
      if (vpre != nullptr)
        ray_load_compact(b, M, v0 >> kRangeSampleBits, v0 & kRangeSampleMask,
                         (v1 >> kRangeSampleBits) - (v0 >> kRangeSampleBits), lane, sv[i]);
      else ray_load(b, M, ray0 + i, lane, sv[i]);
    } else { sv[i][0] = INFINITY; sv[i][1] = INFINITY; }
  }
  // V (loss.py:68,73): samples inside the unit sphere = the finite sdf values.  Counted here, one atomic per segment,
  // instead of by the forward-only tiles (four contended atomics per tile, all tiles of a wave finishing together).
  int nvalid = 0;
#pragma unroll
  for (int i = 0; i < kSegRays; ++i)
    nvalid += __popc(__ballot_sync(0xffffffffu, sv[i][0] != INFINITY)) + __popc(__ballot_sync(0xffffffffu, sv[i][1] != INFINITY));
  if (lane == 0 && nvalid != 0) atomicAdd(b.V_count + o, nvalid);
  int count = 0;
#pragma unroll
  for (int i = 0; i < kSegRays; ++i) {
    if (ray0 + i >= M.n_rays) break;                       // warp-uniform
    bool keep[2]; float de_ds[2]; float res;
    ray_scan_vals(b, th, M, st, ray0 + i, lane, sv[i], keep, de_ds, res);
    count += ray_emit(b, M, st, ray0 + i, lane, keep, de_ds, res, base + count);
  }
  if (lane == 0) seg_cnt[seg_base(M, o) + seg] = count;
}

// exclusive prefix over the object's segment counts -> seg_prefix[0..nseg], band_m[o] = total.  256 threads, named barrier 1.
__device__ inline void scan_prefix(const BatchDev& b, const int* seg_cnt, int* seg_prefix, const int o, const int tid, int* s_wsum) {
  const int lane = tid & 31, warp = tid >> 5;
  const ObjMeta M = b.meta[o];
  const int nseg = (M.n_rays + kSegRays - 1) / kSegRays, sb = seg_base(M, o);
  int carry = 0;
  for (int b0 = 0; b0 < nseg; b0 += 256) {
    const int i = b0 + tid;
    const int v = (i < nseg) ? __ldcg(seg_cnt + sb + i) : 0;
    int x = v;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) { int y = __shfl_up_sync(0xffffffffu, x, d); if (lane >= d) x += y; }
    if (lane == 31) s_wsum[warp] = x;
    asm volatile("bar.sync 1, 256;" ::: "memory");
    int woff = 0, tot = 0;
    for (int w = 0; w < 8; ++w) { if (w < warp) woff += s_wsum[w]; tot += s_wsum[w]; }
    if (i < nseg) seg_prefix[sb + i] = carry + woff + x - v;
    carry += tot;
    asm volatile("bar.sync 1, 256;" ::: "memory");
  }
  if (tid == 0) { seg_prefix[sb + nseg] = carry; b.band_m[o] = carry; }
}

// The per-object scan of the per-iteration schedule: all `nthreads` threads of k_ray_scan's CTA.
// s_cnt: kScanMaxRays ints, s_wsum: 32 ints of shared memory.
__device__ inline void scan_object(const BatchDev& b, const float th, const int o, const int tid, const int nthreads, int* s_cnt,
                                   int* s_wsum) {
  const int lane = tid & 31, warp = tid >> 5, nw = nthreads >> 5;
  const ObjMeta M = b.meta[o];
  ScanState st;
  load_scan_state(b.state[o], st);
  const int N = M.n_rays;
  const bool long_rays = b.D > kLongWin;
  bool keep[2]; float de_ds[2]; float res;
  int nvalid = 0;                                          // (V is counted by the ray-sample tiles on this schedule)
  for (int ray = warp; ray < N; ray += nw) {
    int c;
    if (long_rays) {
      c = long_ray(b, th, M, st, ray, lane, ray * b.D, 0, b.D, false, 0, nvalid);
    } else {
      ray_scan(b, th, M, st, ray, lane, keep, de_ds, res);
      c = __popc(__ballot_sync(0xffffffffu, keep[0])) + __popc(__ballot_sync(0xffffffffu, keep[1]));
    }
    if (lane == 0) s_cnt[ray] = c;
  }
  __syncthreads();
  // block exclusive scan of s_cnt[0..N)
  int carry = 0;
  for (int base = 0; base < N; base += nthreads) {
    const int i = base + tid;
    const int v = (i < N) ? s_cnt[i] : 0;
    int x = v;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) { int y = __shfl_up_sync(0xffffffffu, x, d); if (lane >= d) x += y; }
    if (lane == 31) s_wsum[warp] = x;
    __syncthreads();
    int woff = 0, tot = 0;
    for (int w = 0; w < nw; ++w) { if (w < warp) woff += s_wsum[w]; tot += s_wsum[w]; }
    if (i < N) s_cnt[i] = carry + woff + x - v;
    carry += tot;
    __syncthreads();
  }
  if (tid == 0) b.band_m[o] = carry;
  for (int ray = warp; ray < N; ray += nw) {
    if (long_rays) {
      long_ray(b, th, M, st, ray, lane, ray * b.D, 0, b.D, true, (size_t)M.smp_off + s_cnt[ray], nvalid);
      continue;
    }
    ray_scan(b, th, M, st, ray, lane, keep, de_ds, res);
    ray_emit(b, M, st, ray, lane, keep, de_ds, res, (size_t)M.smp_off + s_cnt[ray]);
  }
}

__global__ void __launch_bounds__(kScanThreads) k_ray_scan(BatchDev b, float th) {
  __shared__ int s_cnt[kScanMaxRays];
  __shared__ int s_wsum[32];
  const int o = blockIdx.x;
  if (b.state[o].status != 0 || b.state[o].mode != DSPGN_MODE_JOINT) return;   // pose-only objects: no render term
  if (b.state[o].n_iter == 0) return;                // a dormant joint slot of a gated run
  scan_object(b, th, o, threadIdx.x, kScanThreads, s_cnt, s_wsum);
}

}  // namespace dspgn
