// A monocular keyframe's detection on the device (mono_sequence.Frame.get_detections, reconstruct/mono_sequence.py:
// 75-114, and the keypoint test of Tracking::GetObjectDetectionsMono, src/Tracking_util.cc:176-201): the largest mask,
// the background pixels of its bbox, undistorted as cv2.undistortPoints does and turned into rays, and the keypoints
// inside the eroded mask.  Float steps are separate _rn operations in numpy's / OpenCV's order, as in dspgn_frame.cuh.
#pragma once
#include <cstdint>

#include "dspgn_frame.cuh"

namespace dspgn {

constexpr int kMonoIters = 5;            // cv2.undistortPoints' default criteria: 5 iterations, no epsilon test
constexpr int kMonoKpPerBlock = 64;      // keypoints per block of the keypoint test (8 per warp)
constexpr int kMonoMaxErosion = 63;

struct MonoParams {
  double P[9];           // the projection after undistortion (P = K), row-major
  double inv_k[9];       // the loader's np.linalg.inv(K)
  double fx, fy, cx, cy, ifx, ify;   // A[0][0], A[1][1], A[0][2], A[1][2], 1./fx, 1./fy as OpenCV takes them
  double k1, k2;
  int img_h, img_w;
  int alpha;             // int(downsample_ratio)
  int erosion;           // Objects.maskErrosion
  int n_masks, n_kp;
  long long mask_stride; // bytes per mask in the staged block (H*W rounded up to 16)
};

// out header (int32): chosen mask, background pixels before subsampling, rays (-1: fewer than 2 pixels), pad
constexpr int kMonoHdr = 4;

// the first mask of largest area (np.argmax of the areas)
__device__ __forceinline__ int mono_largest(const int* area, int n_masks) {
  int best = 0;
  for (int m = 1; m < n_masks; ++m)
    if (area[m] > area[best]) best = m;
  return best;
}

// cvUndistortPointsInternal for distortion (k1, k2, 0, 0, 0), R = I, then P: the fp64 loop in OpenCV's operation
// order, icdist = 1 / (1 + ((k2 r2) + k1) r2) (the numerator and the tangential terms are exactly 1 and 0), with its
// icdist < 0 fallback to the distorted normalised point; returned as float32 like a CV_32FC2 destination.
__device__ __forceinline__ void mono_undistort(const MonoParams& P, double u, double v, float* ou, float* ov) {
  double x = __dmul_rn(__dsub_rn(u, P.cx), P.ifx);
  double y = __dmul_rn(__dsub_rn(v, P.cy), P.ify);
  const double x0 = x, y0 = y;
  for (int j = 0; j < kMonoIters; ++j) {
    const double r2 = __dadd_rn(__dmul_rn(x, x), __dmul_rn(y, y));
    const double icdist = __ddiv_rn(1.0, __dadd_rn(1.0, __dmul_rn(__dadd_rn(__dmul_rn(P.k2, r2), P.k1), r2)));
    if (icdist < 0.0) {
      x = __dmul_rn(__dsub_rn(u, P.cx), P.ifx);
      y = __dmul_rn(__dsub_rn(v, P.cy), P.ify);
      break;
    }
    x = __dmul_rn(x0, icdist);
    y = __dmul_rn(y0, icdist);
  }
  const double xx = __dadd_rn(__dadd_rn(__dmul_rn(P.P[0], x), __dmul_rn(P.P[1], y)), P.P[2]);
  const double yy = __dadd_rn(__dadd_rn(__dmul_rn(P.P[3], x), __dmul_rn(P.P[4], y)), P.P[5]);
  const double ww = __ddiv_rn(1.0, __dadd_rn(__dadd_rn(__dmul_rn(P.P[6], x), __dmul_rn(P.P[7], y)), P.P[8]));
  *ou = __double2float_rn(__dmul_rn(xx, ww));
  *ov = __double2float_rn(__dmul_rn(yy, ww));
}

// ErodedMask(py, px) > 0: every mask pixel of the (2e+1)^2 ellipse of getStructuringElement(MORPH_ELLIPSE) around
// (py, px) that lies inside the image is set (cv::erode's default border ignores the outside).  Row dy spans
// |dx| <= cvRound(e * sqrt((e*e - dy*dy) * (1./(e*e)))); e = 0 is the single pixel.  One warp per keypoint, a lane
// per row.
__device__ __forceinline__ bool mono_inside_eroded(const MonoParams& P, const unsigned char* mk, int py, int px) {
  const int e = P.erosion;
  const double inv_r2 = e ? __ddiv_rn(1.0, (double)(e * e)) : 0.0;
  bool ok = true;
  for (int dy = (int)(threadIdx.x & 31) - e; dy <= e && ok; dy += 32) {
    const int y = py + dy;
    if (y < 0 || y >= P.img_h) continue;
    const int dx = e ? __double2int_rn(__dmul_rn((double)e, __dsqrt_rn(__dmul_rn((double)(e * e - dy * dy), inv_r2)))) : 0;
    const unsigned char* row = mk + (size_t)y * P.img_w;
    const int x1 = min(px + dx, P.img_w - 1);
    for (int x = max(px - dx, 0); x <= x1; ++x)
      if (row[x] == 0) { ok = false; break; }
  }
  return __all_sync(0xffffffffu, ok);
}

// Block 0: the largest mask's background pixels, undistorted, and their rays.  Blocks 1..: kMonoKpPerBlock keypoints
// each, tested against the eroded largest mask; a block writes its count and its passing indices in order.
__global__ void __launch_bounds__(kFrameBoxThreads) k_mono_frame(MonoParams P, const unsigned char* __restrict__ masks,
                                                                 const int* __restrict__ bboxes,
                                                                 const float2* __restrict__ kp,
                                                                 const int* __restrict__ area, int* hdr, float* rays,
                                                                 int* kp_cnt, int* kp_idx) {
  __shared__ int s_w[kFrameBoxThreads / 32];
  __shared__ int s_samp[kFrameBackground][2];
  __shared__ unsigned char s_pass[kMonoKpPerBlock];
  const int m = mono_largest(area, P.n_masks);
  const unsigned char* mk = masks + (size_t)m * P.mask_stride;
  if (blockIdx.x == 0) {
    const int n_bg = frame_background(P, bboxes + 4 * m, mk, s_w, s_samp);
    const int n_s = min(n_bg, kFrameBackground);
    // the reference fails below 2 pixels: cv2.undistortPoints asserts on none, squeeze() leaves 1 pixel 1-D
    if (n_s >= 2) {
      for (int i = threadIdx.x; i < n_s; i += blockDim.x) {
        float fu, fv;
        mono_undistort(P, (double)s_samp[i][0], (double)s_samp[i][1], &fu, &fv);
        const double u = (double)fu, v = (double)fv;
#pragma unroll
        for (int j = 0; j < 3; ++j)
          rays[3 * i + j] = __double2float_rn(
              __dadd_rn(__dadd_rn(__dmul_rn(u, P.inv_k[3 * j]), __dmul_rn(v, P.inv_k[3 * j + 1])), P.inv_k[3 * j + 2]));
      }
    }
    if (threadIdx.x == 0) {
      hdr[0] = m;
      hdr[1] = n_bg;
      hdr[2] = n_s >= 2 ? n_s : -1;
      hdr[3] = 0;
    }
    return;
  }
  const int kb = blockIdx.x - 1;
  const int warp = threadIdx.x >> 5;
  for (int j = warp; j < kMonoKpPerBlock; j += kFrameBoxThreads / 32) {
    const int i = kb * kMonoKpPerBlock + j;
    bool pass = false;
    if (i < P.n_kp) {
      const float2 q = kp[i];
      pass = mono_inside_eroded(P, mk, (int)q.y, (int)q.x);     // cv::Mat::at<float>(pt.y, pt.x) truncates
    }
    if ((threadIdx.x & 31) == 0) s_pass[j] = pass;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    int c = 0;
    for (int j = 0; j < kMonoKpPerBlock; ++j)
      if (s_pass[j]) kp_idx[kb * kMonoKpPerBlock + c++] = kb * kMonoKpPerBlock + j;
    kp_cnt[kb] = c;
  }
}

}  // namespace dspgn
