/* A plain-C caller of the cooperative stop (include/dspgn.h: dspgn_solver_set_stop_flag, DSPGN_ST_STOPPED) in
 * CreateNewMapObjects' shape: LocalMapping registers its `volatile bool mbAbortBA` with the solver once, and another
 * thread (Tracking's InsertKeyFrame, LoopClosing's RequestStop) raises it while LocalMapping waits for the keyframe's
 * objects.  Eigen's column-major strides (row stride 1, column stride rows()).  No Python, no torch.
 *   1. the stereo keyframe (tracked detections gated against the map, one new detection), the flag never raised;
 *   2. the same keyframe, the flag raised by a second pthread `delay_us` after the submit while the wait polls it;
 *      a stopped call creates no object (src/LocalMapping_util.cc:184-185 read literally);
 *   3. the same keyframe again with the flag lowered: the stop of call 2 does not reach it.
 *
 *   keyframe_stop_caller <weights.bin> <input.bin> <output.bin> [delay_us]
 * weights and input as tests/native/keyframe_async_caller.c; output: per call the records, n_vertices, n_faces,
 * vertices and faces, as tests/native/keyframe_mesh_caller.c writes them.
 */
#define _POSIX_C_SOURCE 200809L
#include <pthread.h>
#include <stdbool.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <time.h>
#include "dspgn.h"

#define VOXELS_DIM 16

static volatile bool mbAbortBA = false;   /* LocalMapping's flag: InsertKeyFrame / RequestStop / InterruptBA raise it */
static long g_delay_us = 200;

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

/* the other thread: a new keyframe arrives while the objects are being reconstructed */
static void* insert_keyframe(void* arg) {
  (void)arg;
  struct timespec ts = {0, g_delay_us * 1000L};
  nanosleep(&ts, NULL);
  mbAbortBA = true;
  return NULL;
}

/* one keyframe call, submitted and collected; `raise`: a second thread raises mbAbortBA meanwhile.  Records and meshes
 * appended to `out`; *created: the objects CreateNewMapObjects creates from the call. */
static int call(DspgnSolver* sol, int n, const DspgnObjectIn* in, const int32_t* modes, const DspgnGateIn* gates,
                int raise, FILE* out, int* created, int* stopped) {
  DspgnMeshSpec spec = {VOXELS_DIM, NULL};
  mbAbortBA = false;                                   /* LocalMapping lowers it before it processes a keyframe */
  if (dspgn_keyframe_submit(sol, n, in, modes, gates, &spec)) {
    fprintf(stderr, "keyframe_submit: %s\n", dspgn_last_error());
    return 4;
  }
  pthread_t th;
  if (raise && pthread_create(&th, NULL, insert_keyframe, NULL)) return 6;
  DspgnObjectOut* rec = (DspgnObjectOut*)calloc(n, sizeof(DspgnObjectOut));
  int32_t* nv = (int32_t*)calloc(n, 4);
  int32_t* nf = (int32_t*)calloc(n, 4);
  const int rc = dspgn_keyframe_wait(sol, rec, nv, nf);  /* polls mbAbortBA while it waits */
  if (raise) pthread_join(th, NULL);
  if (rc) { fprintf(stderr, "keyframe_wait: %s\n", dspgn_last_error()); return 4; }
  size_t V = 0, F = 0;
  *stopped = 0;
  for (int i = 0; i < n; ++i) {
    V += nv[i]; F += nf[i];
    if (rec[i].status == DSPGN_ST_STOPPED) ++*stopped;
  }
  *created = 0;
  if (*stopped == 0)                                   /* :184: a stopped call's objects are dropped */
    for (int i = 0; i < n; ++i) *created += rec[i].mesh == DSPGN_MESH_DONE;
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
  if (argc > 4) g_delay_us = atol(argv[4]);
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
  for (int i = 0; i < n; ++i) {
    if (fread(hdr, 4, 3, f) != 3) return 2;
    const int M = hdr[0], N = hdr[1], Nfg = hdr[2];
    float* se3 = rd(f, 16); float* ini = rd(f, 16); float* sim3 = rd(f, 16);
    float* pts = rd(f, (size_t)M * 3); float* rays = rd(f, (size_t)N * 3); float* depth = rd(f, Nfg);
    float* scale = rd(f, 1); float* code = rd(f, 64);
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
  /* LocalMapping's constructor: the flag is registered once, as ORB-SLAM hands it to g2o (setForceStopFlag) */
  if (dspgn_solver_set_stop_flag(sol, (const volatile uint8_t*)&mbAbortBA)) {
    fprintf(stderr, "set_stop_flag: %s\n", dspgn_last_error());
    return 3;
  }
  FILE* out = fopen(argv[3], "wb");
  if (!out) return 2;
  int created[3] = {0, 0, 0}, stopped[3] = {0, 0, 0};
  int rc = 0;
  for (int c = 0; c < 3 && !rc; ++c) rc = call(sol, n + 1, in, modes, gates, c == 1, out, &created[c], &stopped[c]);
  fclose(out);
  if (rc) return rc;
  printf("keyframe_stop_caller: created %d / %d / %d objects, stopped %d / %d / %d\n", created[0], created[1], created[2],
         stopped[0], stopped[1], stopped[2]);
  dspgn_solver_set_stop_flag(sol, NULL);
  dspgn_solver_destroy(sol);
  dspgn_decoder_destroy(dec);
  return 0;
}
