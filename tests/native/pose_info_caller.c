/* A plain-C caller of dspgn_keyframe_batch_gated followed by dspgn_pose_information (include/dspgn.h): the gated
 * keyframe call of keyframe_gate_caller.c, then the information matrix of every record, as the object-camera edges of
 * the joint bundle adjustment would take it (EdgeSE3LieAlgebra::setInformation, src/Optimizer_util.cc:210-217).
 * Matrices are column-major (Eigen: row stride 1, column stride rows()).  No Python, no torch.
 *
 *   pose_info_caller <weights.bin> <input.bin> <output.bin>
 * weights: int32 n_lin, latent, latent_in | per layer: int32 out, in | W[out*in] row-major | b[out]
 * input:   int32 n_det | per detection: int32 M, N, Nfg | SE3Tco[16] | iniSE3Tco[16] | Sim3Tco[16] | pts (M,3) | rays (N,3)
 *          (all col-major) | depth[Nfg] | float scale | code[64]
 * output:  the n_det DspgnObjectOut records | double info[n_det][36] | int32 info_status[n_det]
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
  int n = 0;
  if (!f || fread(&n, 4, 1, f) != 1 || n < 1) return 2;
  DspgnObjectIn* in = (DspgnObjectIn*)calloc(n, sizeof(DspgnObjectIn));
  DspgnGateIn* gates = (DspgnGateIn*)calloc(n, sizeof(DspgnGateIn));
  int32_t* modes = (int32_t*)calloc(n, sizeof(int32_t));
  DspgnObjectOut* out = (DspgnObjectOut*)calloc(n, sizeof(DspgnObjectOut));
  for (int i = 0; i < n; ++i) {
    if (fread(hdr, 4, 3, f) != 3) return 2;
    const int M = hdr[0], N = hdr[1], Nfg = hdr[2];
    float* se3 = rd(f, 16); float* ini = rd(f, 16); float* sim3 = rd(f, 16);
    float* pts = rd(f, (size_t)M * 3); float* rays = rd(f, (size_t)N * 3); float* depth = rd(f, Nfg);
    float* scale = rd(f, 1); float* code = rd(f, 64);
    /* estimate_pose_cam_obj(det->SE3Tco, pMO->scale, det->SurfacePoints, pMO->GetShapeCode()), carrying the rays and
     * depths reconstruct_object(det->Sim3Tco, pts, rays, depth) needs if the check fails */
    in[i].t_cam_obj = se3; in[i].t_rs = 1; in[i].t_cs = 4;
    in[i].pts = pts; in[i].n_pts = M; in[i].pts_rs = 1; in[i].pts_cs = M;
    in[i].rays = rays; in[i].n_rays = N; in[i].rays_rs = 1; in[i].rays_cs = N;
    in[i].depth = depth; in[i].n_depth = Nfg;
    in[i].code = code; in[i].scale = scale[0]; in[i].class_id = 0;
    modes[i] = DSPGN_MODE_POSE;
    gates[i].t_cam_obj_map = ini; gates[i].map_rs = 1; gates[i].map_cs = 4;
    gates[i].t_cam_obj_sim3 = sim3; gates[i].sim3_rs = 1; gates[i].sim3_cs = 4;
    gates[i].gate = 1;                                  /* static map object, Observations() > 2 */
  }
  fclose(f);

  DspgnDecoder* dec = NULL; DspgnSolver* sol = NULL;
  if (dspgn_decoder_create(&spec, W, B, 0, &dec)) { fprintf(stderr, "decoder: %s\n", dspgn_last_error()); return 3; }
  DspgnConfig cfg;
  memset(&cfg, 0, sizeof cfg);                       /* configs/config_kitti.json: optimizer block */
  cfg.k1 = 1.0f; cfg.k2 = 100.0f; cfg.k3 = 0.25f; cfg.k4 = 1e7f; cfg.b1 = 0.2f; cfg.b2 = 0.025f; cfg.lr = 1.0f; cfg.s_damp = 1.0f;
  cfg.num_iterations = 10; cfg.code_len = 64; cfg.num_depth_samples = 50; cfg.cut_off = 0.01f; cfg.pose_only_iterations = 5;
  cfg.sdf_only = 0; cfg.engine = DSPGN_ENGINE_AUTO;
  if (dspgn_solver_create(&cfg, &dec, 1, 0, &sol)) { fprintf(stderr, "solver: %s\n", dspgn_last_error()); return 3; }
  const int rc = dspgn_keyframe_batch_gated(sol, n, in, modes, gates, out);
  if (rc) { fprintf(stderr, "keyframe_batch_gated: %s\n", dspgn_last_error()); return 4; }
  int kept = 0, rejected = 0;
  for (int i = 0; i < n; ++i) {
    if (out[i].gate == DSPGN_GATE_KEPT) ++kept;          /* det->SetPoseMeasurementSE3(out.t_cam_obj) */
    else if (out[i].gate == DSPGN_GATE_REJECTED) ++rejected;   /* det->isNew: a new map object from out.t_cam_obj, out.code */
  }
  /* Eigen::Matrix<double, 6, 6> is column-major; the library's row-major matrices are symmetric, so the same bytes */
  double* info = (double*)calloc((size_t)n * 36, sizeof(double));
  int32_t* info_status = (int32_t*)calloc(n, sizeof(int32_t));
  if (dspgn_pose_information(sol, n, info, info_status)) { fprintf(stderr, "pose_information: %s\n", dspgn_last_error()); return 5; }
  int with_info = 0;
  for (int i = 0; i < n; ++i) with_info += info_status[i] == DSPGN_INFO_OK;
  f = fopen(argv[3], "wb");
  fwrite(out, sizeof(DspgnObjectOut), n, f);
  fwrite(info, sizeof(double), (size_t)n * 36, f);
  fwrite(info_status, sizeof(int32_t), n, f);
  fclose(f);
  printf("pose_info_caller: %d kept, %d rejected, %d with information\n", kept, rejected, with_info);
  dspgn_solver_destroy(sol);
  dspgn_decoder_destroy(dec);
  return 0;
}
