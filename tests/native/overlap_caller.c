/* A plain-C caller with LocalMapping's solver and Tracking's LiDAR frame handle in one process: LocalMapping submits a
 * keyframe's object work (dspgn_keyframe_submit), Tracking builds the next keyframe's detections on the device while
 * it runs (dspgn_lidar_frame_run), then LocalMapping collects (dspgn_keyframe_wait).  While the frame handle is alive
 * the solver's grid-sized launches leave DSPGN_FRAME_RESERVE_SMS SMs free, so the frame call need not wait for the
 * keyframe.  Both are warmed once on the same shapes first.  No Python, no torch.
 *
 *   overlap_caller <weights.bin> <frame.bin> <keyframe.bin> <output.bin>
 * weights:  as c_caller.c
 * frame:    DspgnLidarSpec | int32 n_points, n_boxes, n_masks | scan[n_points*4] | DspgnLidarBox[n_boxes]
 *           | masks[n_masks*img_h*img_w] bytes | bboxes[n_masks*4] int32
 * keyframe: int32 n | per object: int32 M, N, Nfg | T[16] row-major | pts[M*3] | rays[N*3] | depth[Nfg]  (all joint)
 * output:   int32 SM budget of the solver's next launch, int32 keyframe still running when the frame call returned
 *           | DspgnLidarBoxOut[n_boxes] | points | depth | rays | DspgnObjectOut[n]
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
  if (argc < 5) return 2;
  FILE* f = fopen(argv[1], "rb");
  if (!f) return 2;
  int hdr[3];
  if (fread(hdr, 4, 3, f) != 3) return 2;
  DspgnDecoderSpec spec;
  memset(&spec, 0, sizeof spec);
  spec.num_linear = hdr[0]; spec.latent_size = hdr[1]; spec.latent_in_layer = hdr[2];
  const float* W[DSPGN_MAX_LINEAR]; const float* B[DSPGN_MAX_LINEAR];
  for (int k = 0; k < spec.num_linear; ++k) {
    int d[2];
    if (fread(d, 4, 2, f) != 2) return 2;
    spec.out_dim[k] = d[0]; spec.in_dim[k] = d[1];
    W[k] = (const float*)rd(f, 4 * (size_t)d[0] * d[1]); B[k] = (const float*)rd(f, 4 * (size_t)d[0]);
  }
  fclose(f);

  f = fopen(argv[2], "rb");
  if (!f) return 2;
  DspgnLidarSpec ls;
  if (fread(&ls, sizeof ls, 1, f) != 1 || fread(hdr, 4, 3, f) != 3) return 2;
  const int n_points = hdr[0], n_boxes = hdr[1], n_masks = hdr[2];
  const float* scan = (const float*)rd(f, 16 * (size_t)n_points);
  const DspgnLidarBox* boxes = (const DspgnLidarBox*)rd(f, sizeof(DspgnLidarBox) * (size_t)n_boxes);
  const uint8_t* masks = (const uint8_t*)rd(f, (size_t)n_masks * ls.img_h * ls.img_w);
  const int32_t* bboxes = (const int32_t*)rd(f, 16 * (size_t)n_masks);
  fclose(f);

  f = fopen(argv[3], "rb");
  int n = 0;
  if (!f || fread(&n, 4, 1, f) != 1 || n < 1) return 2;
  DspgnObjectIn* in = (DspgnObjectIn*)calloc(n, sizeof(DspgnObjectIn));
  int32_t* modes = (int32_t*)calloc(n, sizeof(int32_t));
  for (int i = 0; i < n; ++i) {
    if (fread(hdr, 4, 3, f) != 3) return 2;
    DspgnObjectIn* o = &in[i];
    o->t_cam_obj = (const float*)rd(f, 64); o->t_rs = 4; o->t_cs = 1;
    o->pts = (const float*)rd(f, 12 * (size_t)hdr[0]); o->n_pts = hdr[0]; o->pts_rs = 3; o->pts_cs = 1;
    o->rays = (const float*)rd(f, 12 * (size_t)hdr[1]); o->n_rays = hdr[1]; o->rays_rs = 3; o->rays_cs = 1;
    o->depth = (const float*)rd(f, 4 * (size_t)hdr[2]); o->n_depth = hdr[2];
    o->scale = 1.f;
    modes[i] = DSPGN_MODE_JOINT;
  }
  fclose(f);

  /* LocalMapping's solver first, then Tracking's frame handle: the budget is read at each launch */
  DspgnDecoder* dec = NULL; DspgnSolver* sol = NULL;
  if (dspgn_decoder_create(&spec, W, B, 0, &dec)) { fprintf(stderr, "decoder: %s\n", dspgn_last_error()); return 3; }
  DspgnConfig cfg;
  memset(&cfg, 0, sizeof cfg);                       /* configs/config_kitti.json: optimizer block */
  cfg.k1 = 1.0f; cfg.k2 = 100.0f; cfg.k3 = 0.25f; cfg.k4 = 1e7f; cfg.b1 = 0.2f; cfg.b2 = 0.025f; cfg.lr = 1.0f; cfg.s_damp = 1.0f;
  cfg.num_iterations = 10; cfg.code_len = 64; cfg.num_depth_samples = 50; cfg.cut_off = 0.01f; cfg.pose_only_iterations = 5;
  if (dspgn_solver_create(&cfg, &dec, 1, 0, &sol)) { fprintf(stderr, "solver: %s\n", dspgn_last_error()); return 3; }
  DspgnLidarFrame* fr = NULL;
  if (dspgn_lidar_frame_create(&ls, 0, &fr)) { fprintf(stderr, "frame: %s\n", dspgn_last_error()); return 3; }
  int32_t budget = 0;
  if (dspgn_debug_sm_budget(sol, 0, &budget)) { fprintf(stderr, "sm_budget: %s\n", dspgn_last_error()); return 4; }

  DspgnLidarBoxOut* bo = (DspgnLidarBoxOut*)malloc(sizeof(DspgnLidarBoxOut) * (n_boxes ? n_boxes : 1));
  DspgnObjectOut* rec = (DspgnObjectOut*)calloc(n, sizeof(DspgnObjectOut));
  /* warm both on the exact shapes (buffers, modules) */
  if (dspgn_lidar_frame_run(fr, scan, n_points, boxes, n_boxes, masks, bboxes, n_masks, bo) ||
      dspgn_keyframe_batch(sol, n, in, modes, rec)) {
    fprintf(stderr, "warm-up: %s\n", dspgn_last_error());
    return 4;
  }
  if (dspgn_keyframe_submit(sol, n, in, modes, NULL, NULL)) { fprintf(stderr, "keyframe_submit: %s\n", dspgn_last_error()); return 4; }
  if (dspgn_lidar_frame_run(fr, scan, n_points, boxes, n_boxes, masks, bboxes, n_masks, bo)) {
    fprintf(stderr, "frame run: %s\n", dspgn_last_error());
    return 4;
  }
  const int32_t running = dspgn_keyframe_query(sol) == 0;
  size_t np_ = 0, nr = 0;
  for (int b = 0; b < n_boxes; ++b) { np_ += bo[b].n_pts; if (bo[b].n_rays > 0) nr += bo[b].n_rays; }
  float* pts = (float*)malloc(12 * (np_ + 1));
  float* depth = (float*)malloc(4 * (np_ + 1));
  float* rays = (float*)malloc(12 * (nr + 1));
  if (dspgn_lidar_frame_results(fr, pts, depth, rays)) { fprintf(stderr, "frame results: %s\n", dspgn_last_error()); return 4; }
  if (dspgn_keyframe_wait(sol, rec, NULL, NULL)) { fprintf(stderr, "keyframe_wait: %s\n", dspgn_last_error()); return 4; }

  f = fopen(argv[4], "wb");
  if (!f) return 2;
  fwrite(&budget, 4, 1, f); fwrite(&running, 4, 1, f);
  fwrite(bo, sizeof(DspgnLidarBoxOut), n_boxes, f);
  fwrite(pts, 12, np_, f); fwrite(depth, 4, np_, f); fwrite(rays, 12, nr, f);
  fwrite(rec, sizeof(DspgnObjectOut), n, f);
  fclose(f);
  printf("overlap_caller: budget %d SMs, %d boxes, %d objects, keyframe running when the frame returned: %d\n", budget,
         n_boxes, n, running);
  dspgn_lidar_frame_destroy(fr);
  dspgn_solver_destroy(sol);
  dspgn_decoder_destroy(dec);
  return 0;
}
