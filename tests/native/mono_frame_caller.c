/* A plain-C caller in the Tracking thread's order (Tracking::GetObjectDetectionsMono, src/Tracking_util.cc:162-207):
 * build a monocular keyframe's detection on the device and test the keyframe's keypoints against the eroded mask in
 * the same call (dspgn_mono_frame_run), then read the background rays and the feature indices.  No Python, no OpenCV.
 *
 *   mono_frame_caller <frame.bin> <output.bin>
 * frame:   DspgnMonoSpec | int32 n_masks, n_kp | masks[n_masks*img_h*img_w] bytes | bboxes[n_masks*4] int32
 *          | keypoints[n_kp*2] float32
 * output:  DspgnMonoOut | int32 is_good | background rays [n_rays*3] | feature indices [n_feature]
 */
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include "dspgn.h"

static void* rd(FILE* f, size_t bytes) {
  void* p = malloc(bytes ? bytes : 1);
  if (bytes && fread(p, 1, bytes, f) != bytes) { fprintf(stderr, "short read\n"); exit(2); }
  return p;
}

int main(int argc, char** argv) {
  if (argc < 3) return 2;
  FILE* f = fopen(argv[1], "rb");
  if (!f) return 2;
  DspgnMonoSpec sp;
  int hdr[2];
  if (fread(&sp, sizeof sp, 1, f) != 1 || fread(hdr, 4, 2, f) != 2) return 2;
  const int n_masks = hdr[0], n_kp = hdr[1];
  const uint8_t* masks = (const uint8_t*)rd(f, (size_t)n_masks * sp.img_h * sp.img_w);
  const int32_t* bboxes = (const int32_t*)rd(f, 16 * (size_t)n_masks);
  const float* kp = (const float*)rd(f, 8 * (size_t)n_kp);
  fclose(f);

  DspgnMonoFrame* fr = NULL;
  if (dspgn_mono_frame_create(&sp, 0, &fr)) { fprintf(stderr, "frame: %s\n", dspgn_last_error()); return 3; }
  DspgnMonoOut out;
  if (dspgn_mono_frame_run(fr, masks, bboxes, n_masks, kp, n_kp, &out)) {
    fprintf(stderr, "frame run: %s\n", dspgn_last_error());
    return 4;
  }
  const int n_rays = out.n_rays > 0 ? out.n_rays : 0;
  float* rays = (float*)malloc(12 * (size_t)(n_rays + 1));
  int32_t* feat = (int32_t*)malloc(4 * (size_t)(out.n_feature + 1));
  if (dspgn_mono_frame_results(fr, rays, feat)) { fprintf(stderr, "frame results: %s\n", dspgn_last_error()); return 4; }
  /* the detection is good iff at least 20 keypoints lie inside the eroded mask */
  const int32_t is_good = out.mask >= 0 && out.n_feature >= 20;

  f = fopen(argv[2], "wb");
  fwrite(&out, sizeof out, 1, f);
  fwrite(&is_good, 4, 1, f);
  fwrite(rays, 12, n_rays, f);
  fwrite(feat, 4, out.n_feature, f);
  fclose(f);
  printf("mono_frame_caller: mask %d, %d rays, %d features\n", out.mask, out.n_rays, out.n_feature);
  dspgn_mono_frame_destroy(fr);
  return 0;
}
