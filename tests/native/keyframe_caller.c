/* A plain-C caller of the C ABI (include/dspgn.h) for the stereo keyframe of src/LocalMapping.cc:88-95: the detections
 * associated with existing map objects (GetNewObservations -> estimate_pose_cam_obj, src/LocalMapping_util.cc:109, with
 * the object's scale and shape code) and the new detections (CreateNewMapObjects -> reconstruct_object, :179, with rays
 * and depths) go into ONE dspgn_keyframe_batch call, one mode per object, with the column-major (Eigen) strides the
 * C++ side holds its matrices in (row stride 1, column stride rows()).  No Python, no torch.
 *
 *   keyframe_caller <weights.bin> <input.bin> <output.bin>
 * weights: int32 n_lin, latent, latent_in | per layer: int32 out, in | W[out*in] row-major | b[out]
 * input:   int32 M, N, Nfg | T[16] col-major | pts col-major | rays col-major | depth | float scale | code[64]
 * output:  the 3 DspgnObjectOut records: tracked (pose of T with the scale divided out), new (T), tracked (flipped pose)
 */
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include "dspgn.h"

static float* rd(FILE* f, size_t n) {
  float* p = (float*)malloc(4 * (n ? n : 1));
  if (n && fread(p, 4, n, f) != n) { fprintf(stderr, "short read\n"); exit(2); }
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
    W[k] = rd(f, (size_t)d[0] * d[1]); B[k] = rd(f, d[0]);
  }
  fclose(f);
  f = fopen(argv[2], "rb");
  if (!f || fread(hdr, 4, 3, f) != 3) return 2;
  const int M = hdr[0], N = hdr[1], Nfg = hdr[2];
  float* T = rd(f, 16); float* pts = rd(f, (size_t)M * 3); float* rays = rd(f, (size_t)N * 3); float* depth = rd(f, Nfg);
  float* scale = rd(f, 1); float* code = rd(f, 64);
  fclose(f);

  DspgnDecoder* dec = NULL; DspgnSolver* sol = NULL;
  if (dspgn_decoder_create(&spec, W, B, 0, &dec)) { fprintf(stderr, "decoder: %s\n", dspgn_last_error()); return 3; }
  DspgnConfig cfg;
  memset(&cfg, 0, sizeof cfg);                       /* configs/config_kitti.json: optimizer block */
  cfg.k1 = 1.0f; cfg.k2 = 100.0f; cfg.k3 = 0.25f; cfg.k4 = 1e7f; cfg.b1 = 0.2f; cfg.b2 = 0.025f; cfg.lr = 1.0f; cfg.s_damp = 1.0f;
  cfg.num_iterations = 10; cfg.code_len = 64; cfg.num_depth_samples = 50; cfg.cut_off = 0.01f; cfg.pose_only_iterations = 5;
  cfg.sdf_only = 0; cfg.engine = DSPGN_ENGINE_AUTO;
  if (dspgn_solver_create(&cfg, &dec, 1, 0, &sol)) { fprintf(stderr, "solver: %s\n", dspgn_last_error()); return 3; }

  /* the tracked detection's pose is SE(3): T with its rotation divided by the object's scale (LocalMapping_util.cc:105-109) */
  float Tse3[16], Tf[16];
  memcpy(Tse3, T, sizeof Tse3);
  for (int c = 0; c < 3; ++c)
    for (int r = 0; r < 3; ++r) Tse3[c * 4 + r] /= scale[0];
  /* a second tracked detection: the same object turned 180 degrees about its y axis (columns 0 and 2 negated) */
  memcpy(Tf, Tse3, sizeof Tf);
  for (int r = 0; r < 4; ++r) { Tf[0 * 4 + r] = -Tse3[0 * 4 + r]; Tf[2 * 4 + r] = -Tse3[2 * 4 + r]; }
  DspgnObjectIn in[3];
  memset(in, 0, sizeof in);
  const int32_t modes[3] = {DSPGN_MODE_POSE, DSPGN_MODE_JOINT, DSPGN_MODE_POSE};
  for (int i = 0; i < 3; ++i) {
    in[i].t_cam_obj = (i == 0) ? Tse3 : (i == 1 ? T : Tf); in[i].t_rs = 1; in[i].t_cs = 4;
    in[i].pts = pts; in[i].n_pts = M; in[i].pts_rs = 1; in[i].pts_cs = M;
    in[i].class_id = 0;
    if (modes[i] == DSPGN_MODE_JOINT) {
      in[i].rays = rays; in[i].n_rays = N; in[i].rays_rs = 1; in[i].rays_cs = N;
      in[i].depth = depth; in[i].n_depth = Nfg; in[i].code = NULL; in[i].scale = 1.f;
    } else {
      in[i].code = code; in[i].scale = scale[0];
    }
  }
  DspgnObjectOut out[3];
  const int rc = dspgn_keyframe_batch(sol, 3, in, modes, out);     /* tracked + new detections, one call */
  if (rc) { fprintf(stderr, "keyframe_batch: %s\n", dspgn_last_error()); return 4; }
  DspgnCounters c;
  dspgn_counters(sol, &c);
  f = fopen(argv[3], "wb");
  fwrite(out, sizeof(DspgnObjectOut), 3, f);
  fclose(f);
  printf("keyframe_caller: status %d/%d/%d kernel launches %lld\n", out[0].status, out[1].status, out[2].status,
         (long long)c.kernel_launches);
  dspgn_solver_destroy(sol);
  dspgn_decoder_destroy(dec);
  return 0;
}
