/* A plain-C caller in the Tracking thread's order (src/Tracking_util.cc:31-57): build a LiDAR keyframe's detections on
 * the device (dspgn_lidar_frame_run), then reconstruct every detection that has rays in ONE dspgn_reconstruct_batch
 * call.  No Python, no torch.
 *
 *   lidar_frame_caller <weights.bin> <frame.bin> <output.bin>
 * weights: as c_caller.c
 * frame:   DspgnLidarSpec | int32 n_points, n_boxes, n_masks | scan[n_points*4] | DspgnLidarBox[n_boxes]
 *          | T_cam_obj[n_boxes][16] row-major | masks[n_masks*img_h*img_w] bytes | bboxes[n_masks*4] int32
 * output:  DspgnLidarBoxOut[n_boxes] | points | depth | rays | per box with rays: int32 status | T[16] | code[64] | loss
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
  if (argc < 4) return 2;
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
  const float* tco = (const float*)rd(f, 64 * (size_t)n_boxes);
  const uint8_t* masks = (const uint8_t*)rd(f, (size_t)n_masks * ls.img_h * ls.img_w);
  const int32_t* bboxes = (const int32_t*)rd(f, 16 * (size_t)n_masks);
  fclose(f);

  DspgnLidarFrame* fr = NULL;
  if (dspgn_lidar_frame_create(&ls, 0, &fr)) { fprintf(stderr, "frame: %s\n", dspgn_last_error()); return 3; }
  DspgnLidarBoxOut* bo = (DspgnLidarBoxOut*)malloc(sizeof(DspgnLidarBoxOut) * (n_boxes ? n_boxes : 1));
  if (dspgn_lidar_frame_run(fr, scan, n_points, boxes, n_boxes, masks, bboxes, n_masks, bo)) {
    fprintf(stderr, "frame run: %s\n", dspgn_last_error());
    return 4;
  }
  size_t np_ = 0, nr = 0;
  for (int b = 0; b < n_boxes; ++b) { np_ += bo[b].n_pts; if (bo[b].n_rays > 0) nr += bo[b].n_rays; }
  float* pts = (float*)malloc(12 * (np_ + 1));
  float* depth = (float*)malloc(4 * (np_ + 1));
  float* rays = (float*)malloc(12 * (nr + 1));
  if (dspgn_lidar_frame_results(fr, pts, depth, rays)) { fprintf(stderr, "frame results: %s\n", dspgn_last_error()); return 4; }

  /* the detections with rays (Tracking keeps every detection; the joint reconstruction needs rays and depth) */
  DspgnObjectIn* in = (DspgnObjectIn*)calloc(n_boxes ? n_boxes : 1, sizeof(DspgnObjectIn));
  int n_obj = 0;
  size_t p0 = 0, r0 = 0;
  for (int b = 0; b < n_boxes; ++b) {
    if (bo[b].n_rays >= 0) {
      DspgnObjectIn* o = &in[n_obj++];
      o->t_cam_obj = tco + 16 * b; o->t_rs = 4; o->t_cs = 1;
      o->pts = pts + 3 * p0; o->n_pts = bo[b].n_pts; o->pts_rs = 3; o->pts_cs = 1;
      o->rays = rays + 3 * r0; o->n_rays = bo[b].n_rays; o->rays_rs = 3; o->rays_cs = 1;
      o->depth = depth + p0; o->n_depth = bo[b].n_pts; o->scale = 1.f;
    }
    p0 += bo[b].n_pts;
    if (bo[b].n_rays > 0) r0 += bo[b].n_rays;
  }
  DspgnDecoder* dec = NULL; DspgnSolver* sol = NULL;
  if (dspgn_decoder_create(&spec, W, B, 0, &dec)) { fprintf(stderr, "decoder: %s\n", dspgn_last_error()); return 3; }
  DspgnConfig cfg;
  memset(&cfg, 0, sizeof cfg);                       /* configs/config_kitti.json: optimizer block */
  cfg.k1 = 1.0f; cfg.k2 = 100.0f; cfg.k3 = 0.25f; cfg.k4 = 1e7f; cfg.b1 = 0.2f; cfg.b2 = 0.025f; cfg.lr = 1.0f; cfg.s_damp = 1.0f;
  cfg.num_iterations = 10; cfg.code_len = 64; cfg.num_depth_samples = 50; cfg.cut_off = 0.01f; cfg.pose_only_iterations = 5;
  if (dspgn_solver_create(&cfg, &dec, 1, 0, &sol)) { fprintf(stderr, "solver: %s\n", dspgn_last_error()); return 3; }
  DspgnObjectOut* out = (DspgnObjectOut*)calloc(n_obj ? n_obj : 1, sizeof(DspgnObjectOut));
  if (n_obj && dspgn_reconstruct_batch(sol, n_obj, in, out)) { fprintf(stderr, "reconstruct_batch: %s\n", dspgn_last_error()); return 4; }

  f = fopen(argv[3], "wb");
  fwrite(bo, sizeof(DspgnLidarBoxOut), n_boxes, f);
  fwrite(pts, 12, np_, f); fwrite(depth, 4, np_, f); fwrite(rays, 12, nr, f);
  for (int i = 0; i < n_obj; ++i) {
    fwrite(&out[i].status, 4, 1, f); fwrite(out[i].t_cam_obj, 4, 16, f); fwrite(out[i].code, 4, 64, f); fwrite(&out[i].loss, 4, 1, f);
  }
  fclose(f);
  printf("lidar_frame_caller: %d boxes, %zu points, %zu rays, %d reconstructed\n", n_boxes, np_, nr, n_obj);
  dspgn_solver_destroy(sol);
  dspgn_decoder_destroy(dec);
  dspgn_lidar_frame_destroy(fr);
  return 0;
}
