/* A plain-C caller of the C ABI (include/dspgn.h) for CreateNewMapObjects with the mesh step batched
 * (src/LocalMapping_util.cc:179-196): one dspgn_reconstruct_batch of the keyframe's new detections -- here the mono
 * path's normal + flipped candidate pair and the detection with its points halved -- then ONE dspgn_mesh_batch of the
 * codes that came back good, instead of one extract_mesh_from_code per object.  No Python, no torch.
 *
 *   mesh_caller <weights.bin> <input.bin> <voxels_dim> <output.bin>
 * weights, input: as c_caller.c
 * output:  int32 n_good | int32 index[n_good] | code[n_good][64] | int32 n_vertices[n_good], n_faces[n_good] |
 *          vertices (f32 x3) | faces (int32 x3), object after object
 */
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include "dspgn.h"

#define N_DET 3

static float* rd(FILE* f, size_t n) {
  float* p = (float*)malloc(4 * (n ? n : 1));
  if (n && fread(p, 4, n, f) != n) { fprintf(stderr, "short read\n"); exit(2); }
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
    W[k] = rd(f, (size_t)d[0] * d[1]); B[k] = rd(f, d[0]);
  }
  fclose(f);
  f = fopen(argv[2], "rb");
  if (!f || fread(hdr, 4, 3, f) != 3) return 2;
  const int M = hdr[0], N = hdr[1], Nfg = hdr[2];
  float* T = rd(f, 16); float* pts = rd(f, (size_t)M * 3); float* rays = rd(f, (size_t)N * 3); float* depth = rd(f, Nfg);
  fclose(f);
  const int dim = atoi(argv[3]);

  DspgnDecoder* dec = NULL; DspgnSolver* sol = NULL;
  if (dspgn_decoder_create(&spec, W, B, 0, &dec)) { fprintf(stderr, "decoder: %s\n", dspgn_last_error()); return 3; }
  DspgnConfig cfg;
  memset(&cfg, 0, sizeof cfg);                       /* configs/config_kitti.json: optimizer block */
  cfg.k1 = 1.0f; cfg.k2 = 100.0f; cfg.k3 = 0.25f; cfg.k4 = 1e7f; cfg.b1 = 0.2f; cfg.b2 = 0.025f; cfg.lr = 1.0f; cfg.s_damp = 1.0f;
  cfg.num_iterations = 10; cfg.code_len = 64; cfg.num_depth_samples = 50; cfg.cut_off = 0.01f; cfg.pose_only_iterations = 5;
  cfg.sdf_only = 0; cfg.engine = DSPGN_ENGINE_AUTO;
  if (dspgn_solver_create(&cfg, &dec, 1, 0, &sol)) { fprintf(stderr, "solver: %s\n", dspgn_last_error()); return 3; }

  float Tf[16];                                      /* flipped candidate, LocalMapping_util.cc:394-401 (col-major) */
  memcpy(Tf, T, sizeof Tf);
  for (int r = 0; r < 4; ++r) { Tf[0 * 4 + r] = -T[0 * 4 + r]; Tf[2 * 4 + r] = -T[2 * 4 + r]; }
  DspgnObjectIn in[N_DET];
  memset(in, 0, sizeof in);
  for (int i = 0; i < N_DET; ++i) {
    in[i].t_cam_obj = i == 1 ? Tf : T; in[i].t_rs = 1; in[i].t_cs = 4;
    in[i].pts = pts; in[i].n_pts = i == 2 ? M / 2 : M; in[i].pts_rs = 1; in[i].pts_cs = M;
    in[i].rays = rays; in[i].n_rays = N; in[i].rays_rs = 1; in[i].rays_cs = N;
    in[i].depth = depth; in[i].n_depth = Nfg; in[i].scale = 1.f;
  }
  DspgnObjectOut out[N_DET];
  if (dspgn_reconstruct_batch(sol, N_DET, in, out)) { fprintf(stderr, "reconstruct_batch: %s\n", dspgn_last_error()); return 4; }

  /* the good codes, contiguous with stride DSPGN_MAX_CODE: exactly the record's code field */
  float codes[N_DET * DSPGN_MAX_CODE];
  int32_t idx[N_DET], nv[N_DET], nf[N_DET];
  int n_good = 0;
  for (int i = 0; i < N_DET; ++i)
    if (out[i].status == DSPGN_ST_OK) { idx[n_good] = i; memcpy(codes + n_good * DSPGN_MAX_CODE, out[i].code, sizeof out[i].code); ++n_good; }
  long long V = 0, F = 0;
  float* verts = NULL; int32_t* faces = NULL;
  if (n_good > 0) {
    if (dspgn_mesh_batch(sol, n_good, codes, DSPGN_MAX_CODE, NULL, dim, nv, nf)) { fprintf(stderr, "mesh_batch: %s\n", dspgn_last_error()); return 5; }
    for (int i = 0; i < n_good; ++i) { V += nv[i]; F += nf[i]; }
    verts = (float*)malloc(12 * (size_t)(V ? V : 1)); faces = (int32_t*)malloc(12 * (size_t)(F ? F : 1));
    if (dspgn_mesh_results(sol, verts, faces, NULL)) { fprintf(stderr, "mesh_results: %s\n", dspgn_last_error()); return 5; }
  }
  DspgnCounters c;
  dspgn_counters(sol, &c);
  f = fopen(argv[4], "wb");
  if (!f) return 2;
  fwrite(&n_good, 4, 1, f); fwrite(idx, 4, n_good, f); fwrite(codes, 4, (size_t)n_good * DSPGN_MAX_CODE, f);
  fwrite(nv, 4, n_good, f); fwrite(nf, 4, n_good, f);
  fwrite(verts, 12, V, f); fwrite(faces, 12, F, f);
  fclose(f);
  printf("mesh_caller: %d of %d detections good, %lld vertices, %lld faces, mesh call: %lld kernel launches\n", n_good, N_DET, V, F,
         (long long)c.kernel_launches);
  free(verts); free(faces);
  dspgn_solver_destroy(sol);
  dspgn_decoder_destroy(dec);
  return 0;
}
