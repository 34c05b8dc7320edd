/* A plain-C caller of dspgn_keyframe_submit / dspgn_keyframe_wait (include/dspgn.h) in LocalMapping::Run's order: the
 * keyframe's object work is submitted first, the mapping steps run on the host while the device works, and the records
 * and meshes are collected before the object bookkeeping.  Eigen's column-major strides (row stride 1, column stride
 * rows()).  No Python, no torch.
 *   1. stereo: the tracked detections gated against the map and one new detection (CreateNewMapObjects);
 *   2. mono: the new detection from its map pose and flipped 180 degrees about y as a pair (ProcessDetectedObjects).
 * Every input array is overwritten with NaN right after the submit: the call must not read it again.
 *
 *   keyframe_async_caller <weights.bin> <input.bin> <output.bin>
 * weights, input and output as tests/native/keyframe_mesh_caller.c.
 */
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include "dspgn.h"

#define VOXELS_DIM 16

static float* rd(FILE* f, size_t n) {
  float* p = (float*)malloc(4 * (n ? n : 1));
  if (n && fread(p, 4, n, f) != n) { fprintf(stderr, "short read\n"); exit(2); }
  return p;
}

static void set_inputs(DspgnObjectIn* o, float* T, int M, int N, int Nfg, float* pts, float* rays, float* depth) {
  o->t_cam_obj = T; o->t_rs = 1; o->t_cs = 4;
  o->pts = pts; o->n_pts = M; o->pts_rs = 1; o->pts_cs = M;
  o->rays = rays; o->n_rays = N; o->rays_rs = 1; o->rays_cs = N;
  o->depth = depth; o->n_depth = Nfg;
}

static void poison(float* p, size_t n) { for (size_t i = 0; i < n; ++i) p[i] = NAN; }

/* the host's own mapping steps (ProcessNewKeyFrame .. SearchInNeighbors) while the device works */
static long mapping_steps(DspgnSolver* sol) {
  volatile double acc = 0.0;
  long polls = 0;
  for (int i = 0; i < 2000000; ++i) acc += (double)i * 1e-9;
  while (dspgn_keyframe_query(sol) == 0) ++polls;       /* never blocks */
  return polls;
}

/* submit, poison the inputs, run the mapping steps, collect; records and meshes appended to `out` */
static int call(DspgnSolver* sol, int n, const DspgnObjectIn* in, const int32_t* modes, const DspgnGateIn* gates,
                const int32_t* pair, float** owned, const size_t* owned_n, int n_owned, FILE* out, int* n_meshes) {
  DspgnMeshSpec spec = {VOXELS_DIM, pair};
  if (dspgn_keyframe_submit(sol, n, in, modes, gates, &spec)) {
    fprintf(stderr, "keyframe_submit: %s\n", dspgn_last_error());
    return 4;
  }
  for (int k = 0; k < n_owned; ++k) poison(owned[k], owned_n[k]);
  DspgnObjectOut probe;
  if (dspgn_results(sol, &probe) != DSPGN_E_BUSY) { fprintf(stderr, "results: not busy in flight\n"); return 5; }
  mapping_steps(sol);
  DspgnObjectOut* rec = (DspgnObjectOut*)calloc(n, sizeof(DspgnObjectOut));
  int32_t* nv = (int32_t*)calloc(n, 4);
  int32_t* nf = (int32_t*)calloc(n, 4);
  if (dspgn_keyframe_wait(sol, rec, nv, nf)) { fprintf(stderr, "keyframe_wait: %s\n", dspgn_last_error()); return 4; }
  size_t V = 0, F = 0;
  for (int i = 0; i < n; ++i) {
    V += nv[i]; F += nf[i];
    if (rec[i].mesh == DSPGN_MESH_DONE) ++*n_meshes;   /* a new MapObject: rec[i].t_cam_obj, rec[i].code and this mesh */
  }
  float* vert = (float*)malloc(12 * (V ? V : 1));
  int32_t* face = (int32_t*)malloc(12 * (F ? F : 1));
  if (dspgn_mesh_results(sol, vert, face, NULL)) { fprintf(stderr, "mesh_results: %s\n", dspgn_last_error()); return 4; }
  fwrite(rec, sizeof(DspgnObjectOut), n, out);
  fwrite(nv, 4, n, out);
  fwrite(nf, 4, n, out);
  fwrite(vert, 12, V, out);
  fwrite(face, 12, F, out);
  free(rec); free(nv); free(nf); free(vert); free(face);
  return 0;
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
  DspgnObjectIn* in = (DspgnObjectIn*)calloc(n + 1, sizeof(DspgnObjectIn));
  DspgnGateIn* gates = (DspgnGateIn*)calloc(n + 1, sizeof(DspgnGateIn));
  int32_t* modes = (int32_t*)calloc(n + 1, sizeof(int32_t));
  float** owned = (float**)calloc(9 * (n + 1), sizeof(float*));
  size_t* owned_n = (size_t*)calloc(9 * (n + 1), sizeof(size_t));
  int n_owned = 0;
#define OWN(p, cnt) (owned[n_owned] = (p), owned_n[n_owned++] = (cnt))
  for (int i = 0; i < n; ++i) {
    if (fread(hdr, 4, 3, f) != 3) return 2;
    const int M = hdr[0], N = hdr[1], Nfg = hdr[2];
    float* se3 = rd(f, 16); float* ini = rd(f, 16); float* sim3 = rd(f, 16);
    float* pts = rd(f, (size_t)M * 3); float* rays = rd(f, (size_t)N * 3); float* depth = rd(f, Nfg);
    float* scale = rd(f, 1); float* code = rd(f, 64);
    OWN(se3, 16); OWN(ini, 16); OWN(sim3, 16); OWN(pts, (size_t)M * 3); OWN(rays, (size_t)N * 3); OWN(depth, Nfg);
    OWN(code, 64);
    set_inputs(&in[i], se3, M, N, Nfg, pts, rays, depth);   /* estimate_pose_cam_obj(det->SE3Tco, ...) */
    in[i].code = code; in[i].scale = scale[0];
    modes[i] = DSPGN_MODE_POSE;
    gates[i].t_cam_obj_map = ini; gates[i].map_rs = 1; gates[i].map_cs = 4;
    gates[i].t_cam_obj_sim3 = sim3; gates[i].sim3_rs = 1; gates[i].sim3_cs = 4;
    gates[i].gate = 1;                                  /* static map object, Observations() > 2 */
  }
  if (fread(hdr, 4, 3, f) != 3) return 2;
  const int M = hdr[0], N = hdr[1], Nfg = hdr[2];
  float* T = rd(f, 16);
  float* pts = rd(f, (size_t)M * 3); float* rays = rd(f, (size_t)N * 3); float* depth = rd(f, Nfg);
  fclose(f);
  /* the mono pair reads its own copies (the stereo call poisons the originals) */
  float* T2 = (float*)malloc(64); float* pts2 = (float*)malloc(12 * (size_t)(M ? M : 1));
  float* rays2 = (float*)malloc(12 * (size_t)(N ? N : 1)); float* depth2 = (float*)malloc(4 * (size_t)(Nfg ? Nfg : 1));
  memcpy(T2, T, 64); memcpy(pts2, pts, 12 * (size_t)M); memcpy(rays2, rays, 12 * (size_t)N); memcpy(depth2, depth, 4 * (size_t)Nfg);
  OWN(T, 16); OWN(pts, (size_t)M * 3); OWN(rays, (size_t)N * 3); OWN(depth, Nfg);
  set_inputs(&in[n], T, M, N, Nfg, pts, rays, depth);   /* reconstruct_object(det->Sim3Tco, pts, rays, depth) */
  modes[n] = DSPGN_MODE_JOINT;

  DspgnDecoder* dec = NULL; DspgnSolver* sol = NULL;
  if (dspgn_decoder_create(&spec, W, B, 0, &dec)) { fprintf(stderr, "decoder: %s\n", dspgn_last_error()); return 3; }
  DspgnConfig cfg;
  memset(&cfg, 0, sizeof cfg);                       /* configs/config_kitti.json: optimizer block */
  cfg.k1 = 1.0f; cfg.k2 = 100.0f; cfg.k3 = 0.25f; cfg.k4 = 1e7f; cfg.b1 = 0.2f; cfg.b2 = 0.025f; cfg.lr = 1.0f; cfg.s_damp = 1.0f;
  cfg.num_iterations = 10; cfg.code_len = 64; cfg.num_depth_samples = 50; cfg.cut_off = 0.01f; cfg.pose_only_iterations = 5;
  cfg.sdf_only = 0; cfg.engine = DSPGN_ENGINE_AUTO;
  if (dspgn_solver_create(&cfg, &dec, 1, 0, &sol)) { fprintf(stderr, "solver: %s\n", dspgn_last_error()); return 3; }
  FILE* out = fopen(argv[3], "wb");
  if (!out) return 2;
  int stereo = 0, mono = 0;
  int rc = call(sol, n + 1, in, modes, gates, NULL, owned, owned_n, n_owned, out, &stereo);
  /* the mono pair: the map pose and the same pose with its x and z axes negated (LocalMapping_util.cc:394-401) */
  DspgnObjectIn pair_in[2];
  set_inputs(&pair_in[0], T2, M, N, Nfg, pts2, rays2, depth2);
  float* Tf = (float*)malloc(64);
  for (int c = 0; c < 4; ++c)
    for (int r = 0; r < 4; ++r) Tf[4 * c + r] = (c == 0 || c == 2) ? -T2[4 * c + r] : T2[4 * c + r];
  pair_in[1] = pair_in[0];
  pair_in[1].t_cam_obj = Tf;
  const int32_t pair[2] = {1, 0};
  float* mono_owned[5] = {T2, Tf, pts2, rays2, depth2};
  const size_t mono_n[5] = {16, 16, (size_t)M * 3, (size_t)N * 3, (size_t)Nfg};
  if (!rc) rc = call(sol, 2, pair_in, NULL, NULL, pair, mono_owned, mono_n, 5, out, &mono);
  fclose(out);
  if (rc) return rc;
  printf("keyframe_async_caller: stereo keyframe %d meshes, mono pair %d meshes\n", stereo, mono);
  dspgn_solver_destroy(sol);
  dspgn_decoder_destroy(dec);
  return 0;
}
