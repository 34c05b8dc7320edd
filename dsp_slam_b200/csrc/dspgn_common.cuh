// Shared device-side structures and small closed forms for libdspgn (sm_90a).
// Reference arithmetic being restated is cited per function (paths relative to the DSP-SLAM repo).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <math.h>
#include "../../include/dspgn.h"

namespace dspgn {

constexpr int kMaxCode = DSPGN_MAX_CODE;       // 64
constexpr int kPInt = 72;                      // internal Jacobian row stride: [code 0..63 | pose 64..70 | pad]
constexpr int kAccStride = kPInt * kPInt + kPInt + 8;  // floats per tile partial: H (upper) | b | {loss_sum, rows, ...}
constexpr int kAccB = kPInt * kPInt;
// H partials are stored as the PACKED upper triangle of the internal 72x72 matrix, row-major: entry (r, c), r <= c, at
// tri_index(r, c) in [0, kTriInt).  The solve reads entry  tid + q*256  -> perfectly coalesced (r*72+c
// addressing would cost one 32-byte sector per lane).
constexpr int kTriInt = kPInt * (kPInt + 1) / 2;
__host__ __device__ __forceinline__ int tri_index(int r, int c) { return r * kPInt - (r * (r - 1)) / 2 + (c - r); }
constexpr int kAccLoss = kAccB + kPInt;        // +0 loss sum, +1 row count
constexpr int kTermSdf = 0, kTermRender = 1;

// Static description of one object of the resident batch.
struct ObjMeta {
  int pts_off, n_pts;          // into pts (xyz interleaved)
  int ray_off, n_rays, n_fg;   // into rays (xyz interleaved); depth_fg offset = fg_off
  int fg_off;
  int smp_off;                 // into per-sample buffers (n_rays * D)
  int class_id;
  float scale;                 // estimate_pose only
  int has_code;
  int bad;                     // unusable detection, rejected at upload: status DSPGN_ST_BAD_INPUT, never evaluated
  int build;                   // device-side input construction: bit 0 rays from pixels (invK), bit 1 world points / world pose (T_cw)
};

// Evolving per-object GN state (device resident for all iterations).
struct ObjState {
  float T_oc[12];              // [R|t] rows, object <- camera (R carries 1/scale)
  float z[kMaxCode];
  float dmin, dmax, dstep, dfar;   // optimizer.py:120-126
  float loss;
  int status;
  int iters;
  int V, m;                    // last render counters
  int n_active;                // pose-only inlier count (optimizer.py:76-78)
  int mode;                    // DSPGN_MODE_JOINT / DSPGN_MODE_POSE, set by k_init for the whole run
  int n_iter;                  // GN iterations this object runs (num_iterations or pose_only_iterations)
  // layer 0 with the latent part folded: zb0[j] = b0[j] + sum_i W0[j][i] z[i]  (i < latent size), refreshed whenever z
  // changes (k_init, end of the solve step).  The tensor-core engine then needs only the 3 xyz columns of layer 0 per
  // point, which it evaluates on the CUDA cores while building the first GEMM operand.
  float zb0[256];
};

// ---- tensor-core engine plan (dspgn_tc.cuh): one entry per GEMM step of a tile -----------------------
constexpr int kTcMaxSteps = 18;
enum { TK_FWD_HIDDEN = 0, TK_FWD_PENULT = 1, TK_BWD_MID = 2, TK_BWD_FIRST = 3 };   // PENULT: last hidden layer + the final Linear(.,1) on the CUDA cores
struct TcStep {
  int kind;
  int n_mma;         // wgmma N of the step: the real output width rounded up to 80, 192 or 256 (tc_mma_n); the
                     // step's weight images hold n_mma rows
  int k_steps;       // K=16 steps of the reduction, a multiple of 4 (whole 64-wide chunks, zero padded)
  int a_reg, d_reg;  // operand / accumulator ping-pong slot of the step (plan bookkeeping)
  unsigned w_off;    // byte offset of this step's first weight image in the blob
  int layer;         // decoder layer (bias / ReLU-mask slot)
  int n_real;        // real output columns (the rest is zero padding)
  int cat_off;       // fwd: K index of the NEXT operand where the decoder input is concatenated; bwd: first
                     // column of the latent_in skip path; -1 = none
  int mask_layer;    // bwd: ReLU mask applied to the outputs; -1 = none
};
struct TcPlan {
  int n_steps, n_fwd;
  TcStep step[kTcMaxSteps];
};

struct SolverParams {
  float k1, k2, k3, k4, b1, b2, lr, s_damp;
  int code_len, D;
  float th;
  int sdf_only;
};

// ---- multi-GPU result exchange (include/dspgn.h "Multi-GPU result exchange") ------------------------------
// All pointers but slot_of point into rank 0's HBM: local memory on rank 0, CUDA-IPC peer mappings (NVLink)
// on every other rank.
struct GatherDev {
  float* slots;          // slot set of this step [n_slots][DSPGN_RESULT_FLOATS]; nullptr = exchange off
  const int* slot_of;    // [n_obj] slot of each resident object (local memory)
  int* flags;            // [world] last step each rank has published
  int* ack;              // last step rank 0 has consumed
  int* err;              // LOCAL error word: 1 = a wait timed out
  long long* wait_ns;    // LOCAL: duration of the last wait (rank 0), for the bench's exchange_ms
  int rank, world, seq;
};

// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ float huber_weight(float a_abs, float b) {
  // loss_utils.py:236-247: w = sqrt(rho)/a; rho = a^2 (a<=b) else 2ba-b^2; a==0 -> 0
  float rho = (a_abs <= b) ? a_abs * a_abs : (2.0f * b * a_abs - b * b);
  float den = (a_abs == 0.0f) ? 1.0f : a_abs;
  return sqrtf(rho) / den;
}

__device__ __forceinline__ float occupancy(float s, float th) {
  // loss_utils.py:40-48
  float c = fminf(fmaxf(s, -th), th);
  return 0.5f - c / (2.0f * th);
}

__device__ __forceinline__ float lin_depth(float dmin, float dmax, float step, int j, int D) {
  // torch.linspace fp32 (optimizer.py:124): symmetric halves, start + step*i as one fused multiply-add
  return (j < D / 2) ? __fmaf_rn(step, (float)j, dmin) : __fmaf_rn(-step, (float)(D - 1 - j), dmax);
}

// Depth samples per ray (DspgnConfig::num_depth_samples) in [2, kMaxDepthSamples].
constexpr int kMaxDepthSamples = 256;
// Range words of the valid-sample hulls (dspgn_solve.cuh: valid_sample_ranges): (row prefix << kRangeSampleBits) | first
// sample.  The field holds every first sample of D <= 256 and leaves 23 bits of prefix for n_rays * D <= 8192 * 256.
constexpr int kRangeSampleBits = 8, kRangeSampleMask = (1 << kRangeSampleBits) - 1;
static_assert(kMaxDepthSamples - 1 <= kRangeSampleMask, "a first sample must fit the range word's sample field");

__device__ __forceinline__ void xform_point(const float* __restrict__ T, float px, float py, float pz,
                                            float& ox, float& oy, float& oz) {
  // loss.py:31-32: products rounded, then summed left to right, then + t (as torch does it)
  ox = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(px, T[0]), __fmul_rn(py, T[1])), __fmul_rn(pz, T[2])), T[3]);
  oy = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(px, T[4]), __fmul_rn(py, T[5])), __fmul_rn(pz, T[6])), T[7]);
  oz = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(px, T[8]), __fmul_rn(py, T[9])), __fmul_rn(pz, T[10])), T[11]);
}

// loss.py:68: a ray sample takes part in the render term when it lies inside the unit sphere.  ONE definition with
// explicit roundings: the tile prologues of both engines and the valid-range pre-pass of the persistent kernel
// (dspgn_solve.cuh: valid_sample_ranges) must take the same decision for the same sample.
__device__ __forceinline__ bool inside_unit_sphere(float x, float y, float z) {
  return sqrtf(__fmaf_rn(z, z, __fmaf_rn(y, y, __fmul_rn(x, x)))) < 1.0f;
}

// 3x4 [A|t] -> inverse [A^-1 | -A^-1 t] (adjugate, fp64 inside, fp32 out)
__device__ inline void inv_affine(const float* T, float* out, double* det_out) {
  double a = T[0], b = T[1], c = T[2], d = T[4], e = T[5], f = T[6], g = T[8], h = T[9], i = T[10];
  double A = e * i - f * h, B = -(d * i - f * g), C = d * h - e * g;
  double det = a * A + b * B + c * C;
  double id = 1.0 / det;
  double m[9] = {A * id, (c * h - b * i) * id, (b * f - c * e) * id,
                 B * id, (a * i - c * g) * id, (c * d - a * f) * id,
                 C * id, (b * g - a * h) * id, (a * e - b * d) * id};
  double tx = T[3], ty = T[7], tz = T[11];
  for (int r = 0; r < 3; ++r) {
    out[r * 4 + 0] = (float)m[r * 3 + 0];
    out[r * 4 + 1] = (float)m[r * 3 + 1];
    out[r * 4 + 2] = (float)m[r * 3 + 2];
    out[r * 4 + 3] = (float)(-(m[r * 3 + 0] * tx + m[r * 3 + 1] * ty + m[r * 3 + 2] * tz));
  }
  if (det_out) *det_out = det;
}

// optimizer.py:120-126: depth range from the current pose.
__device__ inline void derive_depth_range(ObjState& st, int D) {
  float Tco[12];
  double det_oc;
  inv_affine(st.T_oc, Tco, &det_oc);
  float det_co = (float)(1.0 / det_oc);
  float scale = powf(det_co, 1.0f / 3.0f);
  st.dmin = Tco[11] - scale;
  st.dmax = Tco[11] + scale;
  st.dstep = (st.dmax - st.dmin) / (float)(D - 1);
  st.dfar = 1.1f * st.dmax;
}

// loss_utils.py:188-233 (Sim(3)) / 129-163 (SE(3), s ignored, J without scale terms).
__device__ inline void exp_sim3_dev(const float* x, bool sim3, float* out /*3x4*/) {
  float v0 = x[0], v1 = x[1], v2 = x[2], w0 = x[3], w1 = x[4], w2 = x[5];
  float s = sim3 ? x[6] : 0.0f;
  float W[9] = {0.f, -w2, w1, w2, 0.f, -w0, -w1, w0, 0.f};
  float W2[9];
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 3; ++c)
      W2[r * 3 + c] = W[r * 3 + 0] * W[0 * 3 + c] + W[r * 3 + 1] * W[1 * 3 + c] + W[r * 3 + 2] * W[2 * 3 + c];
  float theta = sqrtf(w0 * w0 + w1 * w1 + w2 * w2);
  float th2 = theta * theta;
  float es = sim3 ? expf(s) : 1.0f;
  float R[9], J[9];
  const float I[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1};
  if (theta <= 1e-8f) {
    float c = 1.0f;
    if (sim3 && s != 0.0f) c = (es - 1.0f) / s;
    for (int k = 0; k < 9; ++k) { R[k] = I[k]; J[k] = c * I[k]; }
  } else {
    float sn = sinf(theta), cs = cosf(theta);
    float ra = sn / theta, rb = (1.0f - cs) / th2;
    for (int k = 0; k < 9; ++k) R[k] = I[k] + W[k] * ra + W2[k] * rb;
    if (sim3) {
      float a = es * sn, b = es * cs;
      float c = (s <= 1e-8f) ? 0.0f : (es - 1.0f) / s;      // loss_utils.py:223 quirk kept
      float den = s * s + th2;
      float k1 = (a * s + (1.0f - b) * theta) / den;
      float k2 = c - ((b - 1.0f) * s + a * theta) / den;
      for (int k = 0; k < 9; ++k) J[k] = c * I[k] + (k1 / theta) * W[k] + (k2 / th2) * W2[k];
    } else {
      float k1 = (1.0f - cs) / th2;
      float k2 = (theta - sn) / (th2 * theta);
      for (int k = 0; k < 9; ++k) J[k] = I[k] + k1 * W[k] + k2 * W2[k];
    }
  }
  for (int r = 0; r < 3; ++r) {
    out[r * 4 + 0] = es * R[r * 3 + 0];
    out[r * 4 + 1] = es * R[r * 3 + 1];
    out[r * 4 + 2] = es * R[r * 3 + 2];
    out[r * 4 + 3] = J[r * 3 + 0] * v0 + J[r * 3 + 1] * v1 + J[r * 3 + 2] * v2;
  }
}

// out = A * B for 3x4 affine matrices (implicit last row 0 0 0 1), fp32 like torch.mm
__device__ inline void mul_affine(const float* A, const float* B, float* out) {
  for (int r = 0; r < 3; ++r) {
    for (int c = 0; c < 4; ++c) {
      float acc = A[r * 4 + 0] * B[0 * 4 + c] + A[r * 4 + 1] * B[1 * 4 + c] + A[r * 4 + 2] * B[2 * 4 + c];
      if (c == 3) acc += A[r * 4 + 3];
      out[r * 4 + c] = acc;
    }
  }
}

}  // namespace dspgn
