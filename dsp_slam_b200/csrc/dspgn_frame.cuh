// A KITTI LiDAR keyframe's detection inputs on the device (FrameWithLiDAR.get_detections,
// reconstruct/kitti_sequence.py:99-216): per-box scan point selection, mask association, background pixel sampling
// and rays.  Every value is what numpy computes: float32 / float64 steps as separate _rn operations in numpy's order
// (a 3-term row product is (p0 r0 + p1 r1) + p2 r2, no FMA), and numpy's linspace restated branch by branch.
#pragma once
#include <cstdint>

namespace dspgn {

constexpr int kFrameMaxBoxes = 256;
constexpr int kFrameMaxMasks = 64;
constexpr int kFrameMaxLidar = 4096;
constexpr int kFrameBackground = 200;    // background pixels kept per box (kitti_sequence.py:203-205)
constexpr int kFrameExpand = 5;          // the sampler's crop expansion (:72)
constexpr int kFrameWarps = 4;           // warps per block of the scan passes
constexpr int kFrameChunk = 128;         // scan points per warp chunk (4 rounds of 32)
constexpr int kFrameBoxThreads = 256;

// one box as the device reads it: T_obj_velo rows 0..2, trans, size, front flag (float bits)
constexpr int kFrameBoxWords = 20;

struct FrameParams {
  float K[9];            // row-major
  float inv_k[9];
  float tcv[12];         // T_cam_velo rows 0..2
  int img_h, img_w;
  int num_max;           // num_lidar_max
  int min_area;          // min_mask_area
  int alpha;             // int(downsample_ratio)
  int n_pts, n_boxes, n_masks;
  int n_chunks;
  long long mask_stride; // bytes per mask in the staged block (H*W rounded up to 16)
};

// out header per box (int32): n_pts, n_rays (-1 = None), matched mask (-1 = none), N before subsampling
constexpr int kFrameHdr = 4;

__device__ __forceinline__ float f3dot(float a0, float a1, float a2, float r0, float r1, float r2) {
  return __fadd_rn(__fadd_rn(__fmul_rn(a0, r0), __fmul_rn(a1, r1)), __fmul_rn(a2, r2));
}

// np.linspace(start, stop, num)[i] for integer start / stop (fp64): div = num-1; step = delta/div;
// step == 0 -> (i/div)*delta; div <= 0 -> i*delta; then + start; the last entry is stop when num > 1.
__device__ __forceinline__ double np_linspace(double start, double stop, int num, int i) {
  const double delta = __dsub_rn(stop, start);
  const int div = num - 1;
  double y = (double)i;
  if (div > 0) {
    const double step = __ddiv_rn(delta, (double)div);
    y = (step == 0.0) ? __dmul_rn(__ddiv_rn(y, (double)div), delta) : __dmul_rn(y, step);
  } else {
    y = __dmul_rn(y, delta);
  }
  y = __dadd_rn(y, start);
  if (num > 1 && i == num - 1) y = stop;
  return y;
}

// np.linspace(0, n-1, m).astype(int32) keeps rank r (0 <= r < n, n > m >= 1) at output slot i; -1 if r is not
// kept.  For n > m the step (n-1)/(m-1) exceeds 1, so at most one i truncates to r: i lies in [r/step, (r+1)/step),
// and the candidates around ceil(r/step) are tested with the same fp64 formula.
__device__ __forceinline__ int np_subsample_slot(int r, int n, int m) {
  if (m == 1) return r == 0 ? 0 : -1;
  const double step = __ddiv_rn((double)(n - 1), (double)(m - 1));
  const int c = (int)ceil(__ddiv_rn((double)r, step));
  for (int i = max(c - 1, 0); i <= min(c + 1, m - 1); ++i)
    if ((int)np_linspace(0.0, (double)(n - 1), m, i) == r) return i;
  return -1;
}

__device__ __forceinline__ bool frame_selects(const float* bx, float px, float py, float pz) {
  // the +-3 m cube around trans (x - 3.0 stays float32), then the 1.1-widened box in the object frame
  const float x = bx[12], y = bx[13], z = bx[14];
  if (!(px > __fsub_rn(x, 3.f) && px < __fadd_rn(x, 3.f) && py > __fsub_rn(y, 3.f) && py < __fadd_rn(y, 3.f) &&
        pz > __fsub_rn(z, 3.f) && pz < __fadd_rn(z, 3.f)))
    return false;
  const float hw = __fmul_rn(__fmul_rn(bx[15], 0.5f), 1.1f);
  const float hl = __fmul_rn(__fmul_rn(bx[16], 0.5f), 1.1f);
  const float hh = __fmul_rn(bx[17], 0.5f);
  const float ox = __fadd_rn(f3dot(px, py, pz, bx[0], bx[1], bx[2]), bx[3]);
  const float oy = __fadd_rn(f3dot(px, py, pz, bx[4], bx[5], bx[6]), bx[7]);
  const float oz = __fadd_rn(f3dot(px, py, pz, bx[8], bx[9], bx[10]), bx[11]);
  return ox > -hw && ox < hw && oy > -hh && oy < hh && oz > -hl && oz < hl;
}

// Pass 1 (mode 0) counts each box's selected points per warp chunk into cnt[box][chunk].  Pass 2 (mode 1) reads the
// chunk offsets (cnt after the scan) and writes the kept ranks, in camera frame, to pts[box][slot].
template <int kMode>
__global__ void __launch_bounds__(kFrameWarps * 32) k_frame_select(FrameParams P, const float* __restrict__ boxes,
                                                                   const float4* __restrict__ scan, int* cnt,
                                                                   const int* __restrict__ tot, float* pts) {
  __shared__ float sb[kFrameMaxBoxes * kFrameBoxWords];
  for (int i = threadIdx.x; i < P.n_boxes * kFrameBoxWords; i += blockDim.x) sb[i] = boxes[i];
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const int chunk = blockIdx.x * kFrameWarps + (threadIdx.x >> 5);
  if (chunk >= P.n_chunks) return;
  constexpr int kRounds = kFrameChunk / 32;
  float4 p[kRounds];
  bool ok[kRounds];
#pragma unroll
  for (int k = 0; k < kRounds; ++k) {
    const int i = chunk * kFrameChunk + k * 32 + lane;
    ok[k] = i < P.n_pts;
    p[k] = ok[k] ? scan[i] : make_float4(0.f, 0.f, 0.f, 0.f);
  }
  const unsigned lt = (1u << lane) - 1u;
  for (int b = 0; b < P.n_boxes; ++b) {
    const float* bx = sb + b * kFrameBoxWords;
    int run = 0;
    const int base = kMode ? cnt[(size_t)b * P.n_chunks + chunk] : 0;
    const int N = kMode ? tot[b] : 0;
#pragma unroll
    for (int k = 0; k < kRounds; ++k) {
      const bool sel = ok[k] && frame_selects(bx, p[k].x, p[k].y, p[k].z);
      const unsigned m = __ballot_sync(0xffffffffu, sel);
      if (kMode && sel) {
        const int r = base + run + __popc(m & lt);
        const int slot = (N <= P.num_max) ? r : np_subsample_slot(r, N, P.num_max);
        if (slot >= 0) {
          float* o = pts + ((size_t)b * P.num_max + slot) * 3;
          o[0] = __fadd_rn(f3dot(p[k].x, p[k].y, p[k].z, P.tcv[0], P.tcv[1], P.tcv[2]), P.tcv[3]);
          o[1] = __fadd_rn(f3dot(p[k].x, p[k].y, p[k].z, P.tcv[4], P.tcv[5], P.tcv[6]), P.tcv[7]);
          o[2] = __fadd_rn(f3dot(p[k].x, p[k].y, p[k].z, P.tcv[8], P.tcv[9], P.tcv[10]), P.tcv[11]);
        }
      }
      run += __popc(m);
    }
    if (!kMode && lane == 0) cnt[(size_t)b * P.n_chunks + chunk] = run;
  }
}

// Blocks [0, n_boxes): exclusive scan of one box's chunk counts in place, its total N and n_pts = min(N, num_max)
// into the header.  Blocks [n_boxes, n_boxes + n_masks): one mask's area (nonzero bytes).
__global__ void __launch_bounds__(1024) k_frame_scan_area(FrameParams P, int* cnt, int* tot, int* hdr,
                                                          const unsigned char* __restrict__ masks, int* area) {
  __shared__ int s_w[32];
  __shared__ int s_carry;
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  if ((int)blockIdx.x >= P.n_boxes) {
    const int m = blockIdx.x - P.n_boxes;
    const uint4* src = reinterpret_cast<const uint4*>(masks + (size_t)m * P.mask_stride);
    const long long n16 = P.mask_stride / 16;     // padding bytes are zero
    int c = 0;
    for (long long i = threadIdx.x; i < n16; i += blockDim.x) {
      const uint4 v = src[i];
      c += (__popc(__vcmpne4(v.x, 0u)) + __popc(__vcmpne4(v.y, 0u)) + __popc(__vcmpne4(v.z, 0u)) +
            __popc(__vcmpne4(v.w, 0u))) >> 3;
    }
    c = __reduce_add_sync(0xffffffffu, c);
    if (lane == 0) s_w[w] = c;
    __syncthreads();
    if (threadIdx.x == 0) {
      int a = 0;
      for (int i = 0; i < (int)(blockDim.x >> 5); ++i) a += s_w[i];
      area[m] = a;
    }
    return;
  }
  const int b = blockIdx.x;
  int* c = cnt + (size_t)b * P.n_chunks;
  if (threadIdx.x == 0) s_carry = 0;
  __syncthreads();
  for (int t0 = 0; t0 < P.n_chunks; t0 += blockDim.x) {
    const int i = t0 + threadIdx.x;
    const int v = i < P.n_chunks ? c[i] : 0;
    int x = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int y = __shfl_up_sync(0xffffffffu, x, o);
      if (lane >= o) x += y;
    }
    if (lane == 31) s_w[w] = x;
    __syncthreads();
    if (w == 0) {
      int z = lane < (int)(blockDim.x >> 5) ? s_w[lane] : 0;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const int y = __shfl_up_sync(0xffffffffu, z, o);
        if (lane >= o) z += y;
      }
      s_w[lane] = z;                              // inclusive warp totals
    }
    __syncthreads();
    const int carry = s_carry;
    if (i < P.n_chunks) c[i] = carry + (w ? s_w[w - 1] : 0) + x - v;
    __syncthreads();
    if (threadIdx.x == blockDim.x - 1) s_carry = carry + s_w[(blockDim.x >> 5) - 1];
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    tot[b] = s_carry;
    hdr[b * kFrameHdr + 0] = min(s_carry, P.num_max);
    hdr[b * kFrameHdr + 3] = s_carry;
  }
}

// exclusive block-wide prefix of a per-thread 0/1 flag in scan order; returns the block total
__device__ __forceinline__ int frame_block_rank(bool f, int* s_w, int* rank) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const unsigned m = __ballot_sync(0xffffffffu, f);
  if (lane == 0) s_w[w] = __popc(m);
  __syncthreads();
  int before = 0, total = 0;
  for (int i = 0; i < kFrameBoxThreads / 32; ++i) {
    before += (i < w) ? s_w[i] : 0;
    total += s_w[i];
  }
  *rank = before + __popc(m & ((1u << lane) - 1u));
  __syncthreads();
  return total;
}

// The background sampler of one mask's bbox (kitti_sequence.py:70-92, mono_sequence.py:51-73), for a block of
// kFrameBoxThreads threads: the bbox (l, t, r, b) expanded by 5 px and clamped to the image, the grid
// np.linspace(t, b, int(H/alpha)) x np.linspace(l, r, int(W/alpha)) in row-major order, its pixels outside the mask,
// and, when there are more than 200, the ranks np.linspace(0, n-1, 200).astype(int32).  Writes the kept (u, v) to
// s_samp in order and returns n, the count before subsampling, to every thread.
// Params: FrameParams or MonoParams (img_h, img_w, alpha).
template <class Params>
__device__ __forceinline__ int frame_background(const Params& P, const int* bbox, const unsigned char* mk, int* s_w,
                                                int (*s_samp)[2]) {
  const int max_w = P.img_w - 1, max_h = P.img_h - 1;
  int l = bbox[0], t = bbox[1], r = bbox[2], bt = bbox[3];
  l = l > kFrameExpand ? l - kFrameExpand : 0;
  t = t > kFrameExpand ? t - kFrameExpand : 0;
  r = r < max_w - kFrameExpand ? r + kFrameExpand : max_w;
  bt = bt < max_h - kFrameExpand ? bt + kFrameExpand : max_h;
  const int nh = (bt - t + 1) / P.alpha, nw = (r - l + 1) / P.alpha;    // int(crop / alpha), crop >= 1
  const long long ng = (long long)nh * nw;
  // pass 1: the number of grid pixels outside the mask; pass 2: their ranks, kept by the 200-of-n subsample
  int ns = 0;
  for (long long g = threadIdx.x; g < ng; g += blockDim.x) {
    const int vv = (int)np_linspace((double)t, (double)bt, nh, (int)(g / nw));
    const int uu = (int)np_linspace((double)l, (double)r, nw, (int)(g % nw));
    ns += mk[(size_t)vv * P.img_w + uu] == 0;
  }
  ns = __reduce_add_sync(0xffffffffu, ns);
  if ((threadIdx.x & 31) == 0) s_w[threadIdx.x >> 5] = ns;
  __syncthreads();
  int n_bg = 0;
  for (int i = 0; i < kFrameBoxThreads / 32; ++i) n_bg += s_w[i];
  __syncthreads();
  int base = 0;
  for (long long g0 = 0; g0 < ng; g0 += blockDim.x) {
    const long long g = g0 + threadIdx.x;
    int vv = 0, uu = 0;
    bool f = false;
    if (g < ng) {
      vv = (int)np_linspace((double)t, (double)bt, nh, (int)(g / nw));
      uu = (int)np_linspace((double)l, (double)r, nw, (int)(g % nw));
      f = mk[(size_t)vv * P.img_w + uu] == 0;
    }
    int rank;
    const int tile = frame_block_rank(f, s_w, &rank);
    if (f) {
      const int q = base + rank;
      const int slot = n_bg <= kFrameBackground ? q : np_subsample_slot(q, n_bg, kFrameBackground);
      if (slot >= 0) { s_samp[slot][0] = uu; s_samp[slot][1] = vv; }
    }
    base += tile;
  }
  __syncthreads();
  return n_bg;
}

// the projection of a camera-frame point with K (float32 division; a point behind the camera still yields a value)
__device__ __forceinline__ void frame_project(const FrameParams& P, const float* q, float* u, float* v) {
  const float h0 = f3dot(q[0], q[1], q[2], P.K[0], P.K[1], P.K[2]);
  const float h1 = f3dot(q[0], q[1], q[2], P.K[3], P.K[4], P.K[5]);
  const float h2 = f3dot(q[0], q[1], q[2], P.K[6], P.K[7], P.K[8]);
  *u = __fdiv_rn(h0, h2);
  *v = __fdiv_rn(h1, h2);
}

__device__ __forceinline__ void frame_ray(const FrameParams& P, double u, double v, float* o) {
#pragma unroll
  for (int j = 0; j < 3; ++j)
    o[j] = __double2float_rn(__dadd_rn(__dadd_rn(__dmul_rn(u, (double)P.inv_k[3 * j]), __dmul_rn(v, (double)P.inv_k[3 * j + 1])),
                                       (double)P.inv_k[3 * j + 2]));
}

// One block per box: mask votes of the projected surface points, the first-maximum match, and for a matched mask
// larger than min_mask_area the background sampler, the 200-of-n subsample and the rays.
__global__ void __launch_bounds__(kFrameBoxThreads) k_frame_box(FrameParams P, const float* __restrict__ boxes,
                                                                const float* __restrict__ pts,
                                                                const unsigned char* __restrict__ masks,
                                                                const int* __restrict__ bboxes,
                                                                const int* __restrict__ area, int* hdr, float* rays) {
  __shared__ int s_pix[kFrameMaxLidar];
  __shared__ int s_votes[kFrameMaxMasks];
  __shared__ int s_w[kFrameBoxThreads / 32];
  __shared__ int s_samp[kFrameBackground][2];
  __shared__ int s_kept, s_match;
  const int b = blockIdx.x;
  const int n = hdr[b * kFrameHdr + 0];
  const bool front = __float_as_int(boxes[b * kFrameBoxWords + 18]) != 0;
  if (!front || P.n_masks == 0) {
    if (threadIdx.x == 0) { hdr[b * kFrameHdr + 1] = -1; hdr[b * kFrameHdr + 2] = -1; }
    return;
  }
  const float* bp = pts + (size_t)b * P.num_max * 3;
  if (threadIdx.x == 0) s_kept = 0;
  for (int m = threadIdx.x; m < P.n_masks; m += blockDim.x) s_votes[m] = 0;
  __syncthreads();
  int kept = 0;
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    float u, v;
    frame_project(P, bp + 3 * i, &u, &v);
    const bool in = u > 0.f && u < (float)P.img_w && v > 0.f && v < (float)P.img_h;
    s_pix[i] = in ? (int)v * P.img_w + (int)u : -1;
    kept += in;
  }
  kept = __reduce_add_sync(0xffffffffu, kept);
  if ((threadIdx.x & 31) == 0) atomicAdd(&s_kept, kept);
  __syncthreads();
  for (int m = 0; m < P.n_masks; ++m) {
    const unsigned char* mk = masks + (size_t)m * P.mask_stride;
    int c = 0;
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
      const int q = s_pix[i];
      c += (q >= 0 && mk[q] != 0);
    }
    c = __reduce_add_sync(0xffffffffu, c);
    if ((threadIdx.x & 31) == 0 && c) atomicAdd(&s_votes[m], c);
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    int best = 0;
    for (int m = 1; m < P.n_masks; ++m)
      if (s_votes[m] > s_votes[best]) best = m;
    const int match = (2 * s_votes[best] > s_kept) ? best : -1;      // max > 0.5 * kept (exact for integers)
    hdr[b * kFrameHdr + 2] = match;
    s_match = (match >= 0 && area[match] > P.min_area) ? match : -1;
    if (s_match < 0) hdr[b * kFrameHdr + 1] = -1;
  }
  __syncthreads();
  const int m = s_match;
  if (m < 0) return;
  const int n_bg = frame_background(P, bboxes + 4 * m, masks + (size_t)m * P.mask_stride, s_w, s_samp);
  const int n_s = min(n_bg, kFrameBackground);
  float* ro = rays + (size_t)b * (P.num_max + kFrameBackground) * 3;
  for (int i = threadIdx.x; i < n + n_s; i += blockDim.x) {
    double u, v;
    if (i < n) {
      float fu, fv;
      frame_project(P, bp + 3 * i, &fu, &fv);
      u = (double)fu; v = (double)fv;
    } else {
      u = (double)s_samp[i - n][0]; v = (double)s_samp[i - n][1];
    }
    frame_ray(P, u, v, ro + 3 * i);
  }
  if (threadIdx.x == 0) hdr[b * kFrameHdr + 1] = n + n_s;
}

}  // namespace dspgn
