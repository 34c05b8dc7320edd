/*
 * dspgn.h -- C ABI of libdspgn.so: DSP-SLAM's per-object shape-prior Gauss-Newton reconstruction
 * as hand-written CUDA for NVIDIA H100 (sm_90a).
 *
 * Drop-in boundary.  The reference has no native FFI for this path: its C++ LocalMapping thread
 * calls Python through pybind11 (src/LocalMapping.cc:38-40, src/LocalMapping_util.cc:109-110,
 * 179-181, 390-392), and Python issues PyTorch ops.  The entry points below are what a native
 * binding for exactly those calls binds to; dsp_slam_b200/optimizer.py (ctypes) is that binding,
 * and INTEGRATION.md shows the one-file replacement of reconstruct/optimizer.py.
 *
 *   reference call                                            entry point here
 *   --------------------------------------------------------  -------------------------------
 *   reconstruct.utils.get_decoder (deep_sdf/workspace.py:202)  dspgn_decoder_create
 *   Optimizer.__init__           (reconstruct/optimizer.py:27)  dspgn_solver_create
 *   Optimizer.reconstruct_object (reconstruct/optimizer.py:88)  dspgn_reconstruct_batch
 *   Optimizer.estimate_pose_cam_obj (optimizer.py:45)           dspgn_estimate_pose_batch
 *   one stereo keyframe's two passes (LocalMapping.cc:88-95)     dspgn_keyframe_batch
 *   ... with GetNewObservations' map check (LocalMapping_util.cc:104-147) and the demoted detections'
 *       reconstruction in CreateNewMapObjects (:179)             dspgn_keyframe_batch_gated
 *   ... and the meshes of every object it creates (:179-196), incl. the mono path's map-pose / flipped pair
 *       (ProcessDetectedObjects, :390-428)                       dspgn_keyframe_batch_meshed + dspgn_mesh_results
 *   loss_utils.decode_sdf        (reconstruct/loss_utils.py:51) dspgn_decode_sdf
 *   MeshExtractor.extract_mesh_from_code (optimizer.py:214)     dspgn_mesh_batch + dspgn_mesh_results
 *   the same keyframe call, collected after LocalMapping's own   dspgn_keyframe_submit + dspgn_keyframe_wait
 *       mapping steps (LocalMapping.cc:72-96)
 *   loss.compute_sdf_loss / compute_render_loss (loss.py:22,46) dspgn_debug_system (test hook)
 *
 * Conventions: every function returns 0 on success or a negative DSPGN_E_* code; per-object soft
 * failures (the reference's is_good=False exits, optimizer.py:130-150) are reported in
 * DspgnObjectOut.status and never through the return code; nothing throws across this ABI.
 * All host buffers are caller-owned, plain float32/int32 with explicit element strides (so the
 * column-major arrays pybind11's Eigen casters produce need no host-side transpose); device
 * buffers are owned by the handles.  One solver = one GPU = one host thread at a time.
 */
#ifndef DSPGN_H_
#define DSPGN_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define DSPGN_MAX_CODE 64
#define DSPGN_MAX_LINEAR 12
#define DSPGN_MAX_CLASSES 4
/* SMs a solver's grid-sized launches leave free while a frame handle is alive on its device (dspgn_keyframe_submit) */
#define DSPGN_FRAME_RESERVE_SMS 4

/* return codes */
#define DSPGN_OK 0
#define DSPGN_E_ARG (-1)      /* bad argument / unsupported decoder shape */
#define DSPGN_E_CUDA (-2)     /* CUDA runtime error; see dspgn_last_error() */
#define DSPGN_E_NOGPU (-3)    /* no usable sm_90 device */
#define DSPGN_E_ALLOC (-4)
#define DSPGN_E_PEER (-5)     /* multi-GPU exchange: a peer never published its results (timeout) */
#define DSPGN_E_BUSY (-6)     /* the solver has a submitted call that has not been collected */

/* DspgnObjectOut.status (per-object soft failure = the reference's is_good=False exits) */
#define DSPGN_ST_OK 0
#define DSPGN_ST_SDF_NAN 1     /* optimizer.py:135-136 */
#define DSPGN_ST_RENDER_FEW 2  /* loss.py:72-73 (fewer than 10 samples in the unit sphere) */
#define DSPGN_ST_RENDER_NAN 3  /* optimizer.py:149-150 (no band rows -> NaN loss) */
#define DSPGN_ST_SOLVE 4       /* normal matrix not positive definite / non-finite step */
#define DSPGN_ST_BAD_INPUT 5   /* unusable detection (no surface points, too many rays, ...): never evaluated */
#define DSPGN_ST_STOPPED 6     /* the call was stopped (dspgn_keyframe_stop) before the object's last iteration */

/* kernel schedules of a run (results are bit-identical; the per-iteration schedule exists for debugging / profiling) */
#define DSPGN_SCHED_AUTO 0
#define DSPGN_SCHED_LAUNCHES 1   /* one launch per residual term and solve per GN iteration */
#define DSPGN_SCHED_PERSISTENT 2 /* one persistent object-pipelined kernel for all iterations (every engine) */

/* decoder engines */
#define DSPGN_ENGINE_AUTO 0
#define DSPGN_ENGINE_SIMT 1    /* fp32 FFMA kernels: on-device ground truth */
#define DSPGN_ENGINE_TC 2      /* wgmma tensor-core kernels, 3-pass split-fp16 (fp32-class accuracy) */
/* wgmma tensor-core kernel for plain decoders up to 512 wide (DeepSDF's 8 x 512 network; narrower classes too),
 * both schedules (the persistent one: k_wide_persistent), tensor-core tolerances.  Opt-in only: AUTO never picks it.  Decoders with LayerNorm,
 * xyz_in_all, use_tanh or more than one latent_in layer are refused with DSPGN_E_ARG. */
#define DSPGN_ENGINE_TC_WIDE 3

typedef struct DspgnDecoder DspgnDecoder;
typedef struct DspgnSolver DspgnSolver;

/* A DeepSDF decoder (deep_sdf/deep_sdf_decoder.py:29-63) with weight-norm already folded:
 * layer k is  y = W[k] x + b[k],  W[k] row-major (out_dim[k], in_dim[k]);
 * ReLU after every layer but the last, tanh after the last (deep_sdf_decoder.py:103-108);
 * at layer `latent_in_layer` the (latent_size+3)-wide input is concatenated after the
 * activations (deep_sdf_decoder.py:87-88); -1 = none. */
typedef struct {
  int32_t latent_size;
  int32_t num_linear;
  int32_t in_dim[DSPGN_MAX_LINEAR];
  int32_t out_dim[DSPGN_MAX_LINEAR];
  int32_t latent_in_layer;
  /* Optional variants of deep_sdf_decoder.py (all zero = the plain decoder above):
   *   cat_kind[k]   what is concatenated AFTER the activations at the input of layer k: 0 nothing, 1 the decoder
   *                 input (latent_in, :87-88; several layers allowed), 2 xyz only (xyz_in_all, :89-90).
   *                 latent_in_layer >= 0 is shorthand for cat_kind[latent_in_layer] = 1.
   *   layer_norm[k] 1: LayerNorm (eps 1e-5) between layer k and its ReLU (:58-63,96-102); gamma/beta through
   *                 dspgn_decoder_create_ex
   *   use_tanh      1: an extra tanh on the last layer before the final one (:93-94,107-108)
   * Decoders that use any of them run on the fp32 SIMT engine (the tensor-core engine covers the plain shape). */
  int32_t cat_kind[DSPGN_MAX_LINEAR];
  int32_t layer_norm[DSPGN_MAX_LINEAR];
  int32_t use_tanh;
  int32_t reserved_;
} DspgnDecoderSpec;

/* The `optimizer` block of configs/config_*.json as read by reconstruct/optimizer.py:27-43. */
typedef struct {
  float k1, k2, k3, k4;        /* joint_optim.k1..k4 */
  float b1, b2;                /* Huber thresholds: render, sdf */
  float lr;                    /* joint_optim.learning_rate */
  float s_damp;                /* joint_optim.scale_damping */
  int32_t num_iterations;      /* joint_optim.num_iterations */
  int32_t code_len;            /* 32 or 64 (<= latent_size of the decoders) */
  int32_t num_depth_samples;   /* D, 2..256 (n_rays * D <= 8192 * 256 per object) */
  float cut_off;               /* cut_off_threshold */
  int32_t pose_only_iterations;/* pose_only_optim.num_iterations */
  int32_t sdf_only;            /* 1: skip the render term (BASELINE config 2 "surface-SDF loss") */
  int32_t engine;              /* DSPGN_ENGINE_* */
  int32_t schedule;            /* DSPGN_SCHED_*: 0 = automatic (the persistent kernel, on every engine) */
} DspgnConfig;

/* One detection, host side.  Strides are in elements (floats). */
typedef struct {
  const float* t_cam_obj; int32_t t_rs, t_cs;           /* (4,4) object->camera, Sim(3) */
  const float* pts;  int32_t n_pts;  int32_t pts_rs, pts_cs;    /* (n_pts,3) camera frame */
  const float* rays; int32_t n_rays; int32_t rays_rs, rays_cs;  /* (n_rays,3), foreground first */
  const float* depth; int32_t n_depth;                  /* (n_depth,) foreground depths */
  const float* code;                                    /* (code_len,) initial code or NULL = zeros */
  float scale;                                          /* estimate_pose only: object scale */
  int32_t class_id;                                     /* index into the solver's decoder list */
  /* Optional input construction ON THE DEVICE (SURVEY 8 row f4); all NULL = the arrays above are used as given.
   *   pixels + inv_k   rays[i] = inv_k [u_i, v_i, 1]   (loss_utils.get_rays, reconstruct/loss_utils.py:23-37;
   *                    src/LocalMapping_util.cc:378-386).  (n_rays,2) pixel coordinates replace `rays` (ignored).
   *   t_cam_world      SE(3) world->camera, 4x4 row-major: `pts` are WORLD map points, x_c = R x_w + t
   *                    (LocalMapping_util.cc:344-352), and `t_cam_obj` is the object's WORLD pose T_wo:
   *                    T_co = T_cw T_wo (LocalMapping_util.cc:390). */
  const float* pixels; int32_t pix_rs, pix_cs;
  const float* inv_k;                                   /* 3x3 row-major */
  const float* t_cam_world;                             /* 4x4 row-major */
} DspgnObjectIn;

typedef struct {
  float t_cam_obj[16];            /* row-major (4,4); undefined when status != 0 */
  float code[DSPGN_MAX_CODE];
  float loss;                     /* k1*render + k2*sdf of the last evaluated iteration */
  int32_t status;                 /* DSPGN_ST_* */
  int32_t n_valid;                /* V: ray samples inside the unit sphere, last iteration */
  int32_t n_band;                 /* m: band rows kept, last iteration */
  int32_t iters_done;
  int32_t gate;                   /* dspgn_keyframe_batch_gated: DSPGN_GATE_*; 0 everywhere else */
  union {
    int32_t pad_[2];
    struct {
      int32_t mesh;               /* dspgn_keyframe_batch_meshed: DSPGN_MESH_*; 0 everywhere else */
      int32_t reserved_;
    };
  };
} DspgnObjectOut;                 /* 88 floats */

/* device-side result record (same layout), for callers that keep results on the GPU */
#define DSPGN_RESULT_FLOATS 88

const char* dspgn_last_error(void);
int dspgn_version(void);

int dspgn_decoder_create(const DspgnDecoderSpec* spec, const float* const* W, const float* const* b,
                         int device, DspgnDecoder** out);
/* the same with LayerNorm parameters: ln_gamma[k] / ln_beta[k] (out_dim[k] floats) for layers with layer_norm[k] = 1
 * (entries of other layers are ignored; both arrays may be NULL when no layer is normalised) */
int dspgn_decoder_create_ex(const DspgnDecoderSpec* spec, const float* const* W, const float* const* b,
                            const float* const* ln_gamma, const float* const* ln_beta, int device, DspgnDecoder** out);
void dspgn_decoder_destroy(DspgnDecoder* dec);

int dspgn_solver_create(const DspgnConfig* cfg, DspgnDecoder* const* classes, int n_classes,
                        int device, DspgnSolver** out);
void dspgn_solver_destroy(DspgnSolver* s);
/* stream = a cudaStream_t (NULL = legacy default stream). Work is enqueued on it. */
int dspgn_solver_set_stream(DspgnSolver* s, void* cuda_stream);
int dspgn_solver_engine(const DspgnSolver* s);   /* resolved DSPGN_ENGINE_* */
int dspgn_solver_sync(DspgnSolver* s);           /* wait for everything enqueued on the solver's stream */

/* Whole call, host buffers in, host buffers out (upload + all GN iterations + download + sync). */
int dspgn_reconstruct_batch(DspgnSolver* s, int n_obj, const DspgnObjectIn* in, DspgnObjectOut* out);
int dspgn_estimate_pose_batch(DspgnSolver* s, int n_obj, const DspgnObjectIn* in, DspgnObjectOut* out);

/* The same split into its three phases, for callers that keep a batch resident in HBM:
 *   upload:  pack + H2D of the batch into the solver's workspace (async on the stream)
 *   run:     reset state from the uploaded initial poses/codes, run all GN iterations (async);
 *            mode 0 = joint (reconstruct_object), 1 = pose-only (estimate_pose_cam_obj)
 *   results: D2H + stream sync;  results_device: pointer to n_obj*DSPGN_RESULT_FLOATS floats */
int dspgn_upload_batch(DspgnSolver* s, int n_obj, const DspgnObjectIn* in);
int dspgn_run_batch(DspgnSolver* s, int mode);
int dspgn_results(DspgnSolver* s, DspgnObjectOut* out);
const float* dspgn_results_device(DspgnSolver* s);

/* Per-object run modes: one keyframe's tracked objects (estimate_pose_cam_obj, src/LocalMapping_util.cc:109) and new
 * objects (reconstruct_object, :179) in ONE run.  Every object gets exactly the record the single-mode entry point for
 * its mode writes (pose-only objects: no render term, their rays are ignored; pose_only_iterations iterations).
 * dspgn_run_batch(s, m) is the same run with every mode = m.  A mode outside {0, 1}, or a pose-only object without a
 * code or with scale <= 0, returns DSPGN_E_ARG before anything is enqueued; unusable detections stay per-object
 * DSPGN_ST_BAD_INPUT.  The multi-GPU exchange (dspgn_run_batch_gather) stays single-mode. */
#define DSPGN_MODE_JOINT 0   /* reconstruct_object */
#define DSPGN_MODE_POSE 1    /* estimate_pose_cam_obj */
/* resident batch: modes[i] for uploaded object i (host array of n_obj entries) */
int dspgn_run_batch_modes(DspgnSolver* s, const int32_t* modes);
/* whole call: upload + run + results, walked in resident chunks of 1024 like dspgn_reconstruct_batch */
int dspgn_keyframe_batch(DspgnSolver* s, int n_obj, const DspgnObjectIn* in, const int32_t* modes, DspgnObjectOut* out);

/* The keyframe call with the consistency check of GetNewObservations (src/LocalMapping_util.cc:104-147) on the device,
 * and the joint reconstruction of CreateNewMapObjects (:179) for every tracked detection that fails it, in the same run.
 * For a gated object (gate = 1, mode DSPGN_MODE_POSE) the pose-only estimate Zco -- the record's pose, or the input
 * t_cam_obj after a pose-only soft failure -- is compared with the pose the map predicts, Tco = t_cam_obj_map:
 *   dist2D = |(Zco - Tco) translation x, z| (fp32)  and  e = |log(Tco^-1 Zco)| (SE3Quat, fp64).
 * dist2D < 1 && e < 1.5: out.gate = DSPGN_GATE_KEPT and the record is the pose-only record.  Otherwise the detection is
 * new again: out.gate = DSPGN_GATE_REJECTED and the record is exactly what dspgn_reconstruct_batch returns for the
 * object's DspgnObjectIn with t_cam_obj = t_cam_obj_sim3 and code = NULL (so a gated object carries its rays / depths).
 * The static-object and Observations() > 2 conditions stay with the caller (gate = 0 for the others).  gates = NULL is
 * dspgn_keyframe_batch.  A gate on a joint object, a gate without both matrices, a gate value outside {0, 1} or a gated
 * object with t_cam_world returns DSPGN_E_ARG before anything is enqueued.  A gated object and its joint run occupy two
 * slots of a resident batch of 1024. */
#define DSPGN_GATE_OFF 0        /* not gated */
#define DSPGN_GATE_KEPT 1       /* consistent with the map: the pose-only record */
#define DSPGN_GATE_REJECTED 2   /* inconsistent: the joint record of the detection */
typedef struct {
  const float* t_cam_obj_map;  int32_t map_rs, map_cs;   /* iniSE3Tco = Tcw * Two (SE3), LocalMapping_util.cc:106 */
  const float* t_cam_obj_sim3; int32_t sim3_rs, sim3_cs; /* det->Sim3Tco: the joint run's initial pose */
  int32_t gate;   /* 1: static map object with Observations() > 2 -> apply the check; 0: plain pose-only */
} DspgnGateIn;
int dspgn_keyframe_batch_gated(DspgnSolver* s, int n_obj, const DspgnObjectIn* in, const int32_t* modes,
                               const DspgnGateIn* gates /* n_obj entries, or NULL */, DspgnObjectOut* out);

/* The gated keyframe call that also meshes every object it creates, as CreateNewMapObjects (:179-196) and
 * ProcessDetectedObjects (:390-428) store them: pose, code and mesh from one call.  The records are bit-identical to
 * dspgn_keyframe_batch_gated's with the same arguments, except for out.mesh.  Candidates are the joint objects and the
 * gated objects the device rejects (the mesh of a rejected detection goes to the gated object's index).  A pair
 * (pair[i] = j, pair[j] = i, i < j, both joint) is the mono path's two hypotheses, map pose i and flipped pose j: j wins
 * iff loss[i] > loss[j], whatever the statuses; the loser is DSPGN_MESH_LOST.  A candidate (or a pair's winner) whose
 * status is not DSPGN_ST_OK is DSPGN_MESH_FAILED.  The decision and the grid decode run on the device after the last
 * GN iteration, in the run's own resident batch; every DSPGN_MESH_DONE mesh is bit-identical to dspgn_mesh_batch of
 * the record's code and class_id at the same voxels_dim on the same engine.  dspgn_mesh_results then returns the meshes
 * object after object over all n_obj objects (0 vertices / faces without a mesh) and n_obj x dim^3 grids (NaN for
 * objects without one).  modes = NULL: every object joint.  A bad voxels_dim, a pair on a pose-only or gated object, or
 * a pair array that is not symmetric, pairs an object with itself or points out of range returns DSPGN_E_ARG before
 * anything is enqueued.  Counters: rows_fwd_only += dim^3 per meshed object; the mesh launches are counted. */
#define DSPGN_MESH_OFF 0      /* not a mesh candidate (pose-only record, kept gated object) */
#define DSPGN_MESH_DONE 1     /* the object's mesh is in this call's dspgn_mesh_results */
#define DSPGN_MESH_FAILED 2   /* candidate whose record has status != DSPGN_ST_OK: no mesh (CreateNewMapObjects skips it) */
#define DSPGN_MESH_LOST 3     /* the other hypothesis of its pair has the lower loss: no mesh */
typedef struct {
  int32_t voxels_dim;         /* 2..128, as dspgn_mesh_batch */
  const int32_t* pair;        /* n_obj entries or NULL: pair[i] = j and pair[j] = i make joint objects i < j the two
                                 hypotheses of one mono detection (i = map pose, j = flipped); -1 = unpaired */
} DspgnMeshSpec;
int dspgn_keyframe_batch_meshed(DspgnSolver* s, int n_obj, const DspgnObjectIn* in, const int32_t* modes /* or NULL */,
                                const DspgnGateIn* gates /* or NULL */, const DspgnMeshSpec* mesh, DspgnObjectOut* out,
                                int32_t* n_vertices, int32_t* n_faces /* n_obj entries each */);

/* The meshed (or gated) keyframe call without blocking the calling thread: submit a keyframe's object work, do other
 * work (LocalMapping's own mapping steps), collect the records and meshes afterwards.
 *   submit  validates, packs every input into the solver's pinned staging, enqueues the upload, the run, the mesh passes
 *           and asynchronous copies of the records, the mesh counts and the meshes into pinned memory, records an event
 *           and returns.  It never waits for the device once the solver's buffers are large enough for the keyframe
 *           (a call that grows one frees the old buffer, which waits).  Every input array may be freed or overwritten as
 *           soon as it returns.  Arguments as dspgn_keyframe_batch_meshed; mesh = NULL is dspgn_keyframe_batch_gated,
 *           modes = NULL: every object joint.  Scope: one resident chunk -- at most 1024 slots (a gated object takes
 *           two) and at most 2^24 candidate grid rows (64 objects at 64^3); a larger keyframe returns DSPGN_E_ARG (the
 *           blocking calls take any size).
 *   query   1 when the submitted call has finished, 0 while it runs, < 0 on error; never blocks.
 *   wait    blocks until the call has finished and writes what the blocking call writes: n_obj records, and with a mesh
 *           spec n_vertices / n_faces (NULL iff the submit had no mesh spec); dspgn_mesh_results then returns the
 *           meshes.  Records, counts and meshes are bit-identical to dspgn_keyframe_batch_meshed / _gated.
 * One call in flight per solver: until wait, every other entry point on the solver returns DSPGN_E_BUSY (results_device
 * and gather_device return NULL, gather_close does nothing) and leaves the call intact, except query, wait,
 * dspgn_keyframe_stop, dspgn_solver_sync, dspgn_solver_engine and dspgn_debug_host_syncs; dspgn_solver_destroy waits for
 * the call first.
 * Solvers on different streams may each have a call in flight.  The multi-GPU exchange does not apply.
 * SM budget: the persistent kernels fill a whole SM per CTA, so while one runs on every SM no block of another kernel
 * starts anywhere.  While at least one frame handle (DspgnLidarFrame, DspgnMonoFrame) is alive on the solver's device,
 * every grid-sized launch of every solver there -- the persistent kernels and the per-iteration schedule's decoder
 * launches, of this call and of the blocking ones -- uses DSPGN_FRAME_RESERVE_SMS fewer CTAs than the device has SMs,
 * so a Tracking thread's frame call runs beside the keyframe instead of after it.  The budget is read at each launch
 * (a frame handle may be created after the solver); with no frame handle the launches use every SM.  Records and
 * meshes do not depend on the budget: they are bit-identical at every SM count. */
int dspgn_keyframe_submit(DspgnSolver* s, int n_obj, const DspgnObjectIn* in, const int32_t* modes /* or NULL: all joint */,
                          const DspgnGateIn* gates /* or NULL */, const DspgnMeshSpec* mesh /* or NULL */);
int dspgn_keyframe_query(DspgnSolver* s);
int dspgn_keyframe_wait(DspgnSolver* s, DspgnObjectOut* out, int32_t* n_vertices, int32_t* n_faces);
/* The pose information of every record of the solver's last completed call that returned records --
 * dspgn_reconstruct_batch, dspgn_estimate_pose_batch, dspgn_keyframe_batch, _gated, _meshed or dspgn_keyframe_wait --
 * in the call's object order (both hypotheses of a mono pair, every chunk of a call longer than 1024 objects), for the
 * object-camera edges of DSP-SLAM's joint bundle adjustment (EdgeSE3LieAlgebra, measurement det->SE3Tco).
 * Every solve keeps its object's normal matrix H without the damping (the code and rotation priors included); for each
 * record this takes H of the iteration the record's pose came from (a stopped object: its last completed iteration; a
 * gated object: the pose-only solve when KEPT, the joint run's when REJECTED), eliminates scale and code (Schur
 * complement, fp64), and maps the 6x6 result from the solver's left perturbation of T_obj_cam into the edge's tangent
 * space: e = [omega, upsilon] (g2o SE3Quat::log order) with the perturbed pose Z exp(e), Z = the record's pose with its
 * scale divided out of the rotation (SetPoseMeasurementSim3 / SE3).  DESIGN.md §4.13 derives the map.
 *   info         n x 36 doubles, row-major 6x6 per object, in the units of the system the record came from: a joint
 *                record's residuals are row means weighted by k1 (render) and k2 (SDF), plus the code and rotation
 *                priors (optimizer.py:155-184); a pose-only record's are the plain SDF row mean, no k2 and no prior
 *                (optimizer.py:68-70).  Multiply a pose-only record's info by k2 to put it on the joint records' scale;
 *   info_status  DSPGN_INFO_OK, or DSPGN_INFO_NONE (zeros in info): the record has no valid linearisation (status not
 *                DSPGN_ST_OK / DSPGN_ST_STOPPED, or no completed iteration), or the marginal system is not positive
 *                definite.
 * n must equal the call's object count; after a call without records (mesh, decode, the split-phase and multi-GPU runs)
 * or before any call: DSPGN_E_ARG.  DSPGN_E_BUSY while a submitted call is in flight.  Never part of the calls above:
 * it enqueues one kernel and its copies of its own and waits for them. */
#define DSPGN_INFO_OK 0
#define DSPGN_INFO_NONE 1
int dspgn_pose_information(DspgnSolver* s, int n, double* info /* n x 36, row-major */, int32_t* info_status /* n */);
/* Debug: the number of times the solver's calls have blocked the calling thread on the device so far (stream and event
 * synchronisations, counted only when the device still had work to finish). */
int dspgn_debug_host_syncs(DspgnSolver* s, int64_t* out);

/* Cooperative stop of a running keyframe call: LocalMapping's mbAbortBA (src/LocalMapping.cc:165-170, :611, :680), which
 * CreateNewMapObjects checks before and after each reconstruct_object (src/LocalMapping_util.cc:168-169, 184-185) and
 * ORB-SLAM hands to g2o as its force-stop flag.
 *   stoppable objects  the joint objects of dspgn_reconstruct_batch and of the keyframe calls (blocking and submitted),
 *                      including the joint slot of a gated object, except both hypotheses of a mono pair.  Pose-only
 *                      objects, pairs and the multi-GPU exchange always run to the end.
 *   when               a stoppable object reads the stop word once in each solve that is not its last; observed, the
 *                      stop takes effect after that iteration's update: the object finishes with status
 *                      DSPGN_ST_STOPPED (a solve that fails keeps its own status), and its record -- status
 *                      word aside -- is bit-identical to the record of the same call with num_iterations = iters_done.
 *                      Every other record is the unstopped call's.
 *   gated objects      the pose-only record and its gate word are always complete.  A REJECTED object whose joint slot
 *                      would wake after the stop was observed does not run it: its record is DSPGN_ST_STOPPED with
 *                      iters_done 0, pose t_cam_obj_sim3, code zero, loss / n_valid / n_band 0, gate DSPGN_GATE_REJECTED.
 *   meshes             a STOPPED candidate is DSPGN_MESH_FAILED (its grid NaN); every other mesh is the unstopped call's.
 *   return codes       a stopped call returns DSPGN_OK; counters count the rows of the iterations that ran.
 * dspgn_keyframe_stop  requests the stop of the solver's call in flight (dspgn_reconstruct_batch, dspgn_keyframe_batch*,
 *                      or a submitted call until its wait returns).  Nothing in flight: no effect -- a stop never reaches a
 *                      later call (each call has its own generation, which the kernels compare with the stop word).  The one
 *                      entry point that may be called from any thread while another thread is inside a call on the same
 *                      solver (never concurrently with dspgn_solver_destroy); it never blocks and never touches the stream.
 * dspgn_solver_set_stop_flag  registers a caller-owned byte (a C++ bool such as &mbAbortBA; NULL unregisters): while a
 *                      call waits for the device (the blocking calls' synchronisations, dspgn_keyframe_wait) it polls the
 *                      byte between cudaEventQuery polls (yielding the core, never a timed sleep), and a nonzero value becomes
 *                      dspgn_keyframe_stop.  Each such wait counts as one host sync.  No flag: every wait is a plain
 *                      blocking synchronisation, as before. */
int dspgn_keyframe_stop(DspgnSolver* s);
int dspgn_solver_set_stop_flag(DspgnSolver* s, const volatile uint8_t* flag);
/* Test hook: in the next stoppable call the device raises that call's stop itself in caller object `obj`'s solve of
 * iteration `iter` (0-based), just before that solve reads the stop word: a stoppable object then ends STOPPED
 * with iters_done = iter + 1; a pose-only object raises it after any of its iterations, its last included (a gated one
 * before its verdict wakes the joint slot).  A stoppable object's last solve reads nothing and raises nothing.  -1, -1
 * clears it; anything else out of range returns DSPGN_E_ARG. */
int dspgn_debug_stop_at(DspgnSolver* s, int obj, int iter);
/* Test hook: the mesh arena of the following submits holds max_vertices vertices and max_faces faces (both 0: the
 * automatic size, a per-object estimate that grows with the meshes the solver has seen).  A keyframe whose meshes do not
 * fit is meshed again at the exact size inside dspgn_keyframe_wait: slower, never different. */
int dspgn_debug_mesh_arena(DspgnSolver* s, int64_t max_vertices, int64_t max_faces);
/* Test hook: the SM budget of the solver's grid-sized launches (dspgn_keyframe_submit).  n = 0 restores the automatic
 * budget, 1 <= n <= the device's SM count forces n SMs, anything else returns DSPGN_E_ARG.  current (may be NULL)
 * receives the SM count the next grid-sized launch would use. */
int dspgn_debug_sm_budget(DspgnSolver* s, int n, int32_t* current);

/* Forward-only decode (loss_utils.decode_sdf): x (n,3) host, strides in elements -> sdf (n,) host. */
int dspgn_decode_sdf(DspgnSolver* s, int class_id, const float* code, const float* x, int n,
                     int x_rs, int x_cs, float* sdf_out);

/* MeshExtractor.extract_mesh_from_code (reconstruct/optimizer.py:214-223) for n codes at once, on the device: the
 * voxels_dim^3 grid of create_voxel_grid (written on the device) decoded like dspgn_decode_sdf, then the iso-surface
 * sdf = 0 by marching tetrahedra, bit-identical in vertex and face order to dsp_slam_b200/mesh.py's
 * marching_tetrahedra(grid, 0, h = 2/(dim-1)) with every vertex shifted by -1 as extract_mesh_from_code does.
 * Replaces the solver's resident batch (like dspgn_decode_sdf).  codes: n x code_stride floats, the first code_len
 * used.  class_ids NULL = class 0.  2 <= voxels_dim <= 128, else DSPGN_E_ARG; misuse returns DSPGN_E_ARG before anything
 * is enqueued.  Objects are meshed in chunks of at most 2^24 grid rows; the grids of the call stay in HBM.
 * Counters: rows_fwd_only += n * dim^3, and the call's launches. */
int dspgn_mesh_batch(DspgnSolver* s, int n, const float* codes, int code_stride, const int32_t* class_ids,
                     int voxels_dim, int32_t* n_vertices, int32_t* n_faces);
/* the meshes of the last mesh call, object after object: vertices (sum n_vertices x 3, f32, object frame),
 * faces (sum n_faces x 3, int32, indices local to the object's own vertices), sdf (n x dim^3, may be NULL) */
int dspgn_mesh_results(DspgnSolver* s, float* vertices, int32_t* faces, float* sdf);
/* test hook: the same iso-surface on n caller-given grids (n x dim^3 host floats) */
int dspgn_debug_mesh_grid(DspgnSolver* s, int n, int voxels_dim, const float* sdf, int32_t* n_vertices, int32_t* n_faces);

/* Counters of the last run (for roofline arithmetic): decoder rows evaluated fwd+bwd (SDF rows + band rows) and
 * fwd-only, and the number of kernel launches issued.  Persistent schedule: fwd-only rows = the sum of V over objects
 * and iterations, i.e. the ray samples inside the unit sphere, which is what the reference decodes (loss.py:68,77-78);
 * one-launch-per-term schedule: every n_rays x D sample it evaluates. */
typedef struct {
  int64_t rows_fwd_bwd;
  int64_t rows_fwd_only;
  int64_t kernel_launches;
  float decoder_ms;      /* device time of the decoder kernels of the last run (CUDA events), if timed */
  float total_ms;
  float solve_ms;        /* device time of the per-object solve kernels of the last run, if timed */
  float pad_;
} DspgnCounters;
int dspgn_counters(DspgnSolver* s, DspgnCounters* out);
int dspgn_enable_timing(DspgnSolver* s, int on);

/* ---- Multi-GPU result exchange (SURVEY 8e; the reference reconstructs objects one by one on one GPU,
 * src/LocalMapping_util.cc:165-203 -- objects are independent, so a batch is sharded object-per-GPU).
 * One process per GPU.  There is no collective kernel: rank 0 owns a "gather buffer" in its HBM, exports it
 * with CUDA IPC, every other rank maps it over NVLink/NVSwitch, and the solve step that finishes an object
 * stores the object's 352-byte result record STRAIGHT INTO rank 0's buffer (peer st.global issued from the
 * same kernel that runs the tensor-core tiles), at the object's slot = its index in the original batch.  A
 * per-rank sequence flag (release, system scope) publishes a finished step; rank 0 waits for all flags with
 * a one-warp kernel on its own stream.  Two slot sets alternate by step parity and rank 0 acknowledges
 * consumed steps, so ranks may run at most one step ahead of rank 0.  `seq` = 1, 2, 3, ... (caller-owned,
 * identical on all ranks).
 *   rank 0:   gather_create -> (handle to the peers by any host channel) ;  ranks 1..: gather_open
 *   per step, every rank:  upload_batch ; gather_bind(slots) ; run_batch_gather(mode, seq)
 *   rank 0:   gather_results(seq, n, out)  (D2H + sync)   or   gather_device(seq) to keep them in HBM */
#define DSPGN_IPC_HANDLE_BYTES 64
typedef struct { unsigned char bytes[DSPGN_IPC_HANDLE_BYTES]; } DspgnIpcHandle;
int dspgn_gather_create(DspgnSolver* s, int n_slots, int world, DspgnIpcHandle* handle_out);
int dspgn_gather_open(DspgnSolver* s, const DspgnIpcHandle* handle, int n_slots, int world, int rank);
/* slots[i] = slot of resident object i (n == resident objects); n == 0: this rank owns no object this step */
int dspgn_gather_bind(DspgnSolver* s, const int32_t* slots, int n);
int dspgn_run_batch_gather(DspgnSolver* s, int mode, int seq);
int dspgn_gather_results(DspgnSolver* s, int seq, int n, DspgnObjectOut* out);
const float* dspgn_gather_device(DspgnSolver* s, int seq);
/* device time the root's wait kernel spent spinning in the last run_batch_gather (ns, after a sync); -1 if n/a */
long long dspgn_gather_wait_ns(DspgnSolver* s);
void dspgn_gather_close(DspgnSolver* s);

/* Test hook: Lie-group exponentials exactly as the solve step applies them (loss_utils.py:129-233):
 * x (n,7) -> out (n,12) row-major 3x4 [sR | J v]; sim3 = 0 ignores x[6] (exp_se3). */
int dspgn_debug_exp(int device, int sim3, const float* x, int n, float* out);

/* Test hook: evaluate one GN iteration at the uploaded initial state of object `obj` WITHOUT
 * updating it and return the assembled system: H (P*P row-major), b (P), dx (P), P = 7+code_len
 * (mode 0) or 6 (mode 1); J_rows/res_rows (may be NULL): the SDF-term Jacobian rows (n_pts,P) and
 * residuals (n_pts) as loss.compute_sdf_loss returns them. */
int dspgn_debug_system(DspgnSolver* s, int obj, int mode, float* H, float* b, float* dx,
                       float* J_rows, float* res_rows, float* losses /* [sdf, render, V, m] */);
/* The same after advancing the uploaded batch `iter` GN iterations from its initial state (iter = 0: identical
 * to dspgn_debug_system): the system the (iter+1)-th iteration solves, for iteration-by-iteration parity
 * against the reference's captured H/b/dx of every iteration (tests/golden/recon_*.npz H_iters[iter]). */
int dspgn_debug_system_iter(DspgnSolver* s, int obj, int mode, int iter, float* H, float* b, float* dx,
                            float* J_rows, float* res_rows, float* losses);

/* Test hook for the device-side input construction: the resident batch's object `obj` as the kernels see it --
 * t_cam_obj (16, row-major), pts (n_pts*3, xyz interleaved), rays (n_rays*3).  Any pointer may be NULL. */
int dspgn_debug_inputs(DspgnSolver* s, int obj, float* t_cam_obj, float* pts, float* rays);

/* Debug: event log of the last persistent-kernel run (tile begin/end per kind, scan, solve, queue pops), enabled by
 * env DSPGN_CLK at solver creation; returns the number of (timestamp, descriptor) pairs written, or a negative code.
 * out[2i] = %globaltimer (ns), out[2i+1] = kind<<56 | mode<<52 | sm<<40 | object<<24 | tile (or iteration, solve phase);
 * tools/mega_timeline.py decodes it. */
int dspgn_debug_events(DspgnSolver* s, long long* out, int max_events);

/* ---- A KITTI LiDAR keyframe's detections (FrameWithLiDAR.get_detections, reconstruct/kitti_sequence.py:99-216),
 * built on the device from the raw scan, the 3D boxes and the 2D masks.  Its own handle: Tracking builds detections
 * in another thread than LocalMapping's solver calls (src/Tracking_util.cc:31-57), and a solver is one host thread.
 * Per box (the caller keeps the boxes in depth order, np.argsort(detections_3d[:, 0])):
 *   points  the scan points with x-3 < px < x+3 on all three axes (float32), transformed by t_obj_velo and strictly
 *           inside +-1.1 w/2, +-h/2, +-1.1 l/2, in scan order; more than num_lidar_max of them are subsampled at the
 *           ranks np.linspace(0, N-1, num_lidar_max).astype(int32); then transformed by T_cam_velo.
 *   mask    front boxes of a frame with masks: the points projected with K (float32 division), the pixels strictly
 *           inside the image truncated to int, one vote per pixel per mask containing it; the first mask with the
 *           most votes matches iff votes > 0.5 * (pixels inside).
 *   rays    a matched mask with area > min_mask_area: the background grid of its bbox (truncated, expanded by 5 px,
 *           clamped; np.linspace(t, b, int(H/alpha)) x np.linspace(l, r, int(W/alpha)), row-major) outside the mask,
 *           200 of them at np.linspace(0, n-1, 200) ranks when more, appended to the projected (u, v) of every point
 *           (including those outside the image); rays = inv_k [u, v, 1] in float64, cast to float32.  depth = z.
 * Every float step is rounded as numpy rounds it, so the arrays are bit-identical to the reference's.
 *   run      validates (DSPGN_E_ARG before anything is enqueued), stages the scan and the masks in pinned memory, one
 *            H2D copy, four kernels and one D2H copy on the handle's stream, then waits for that copy (the only host
 *            synchronisation) and writes one DspgnLidarBoxOut per box.  Limits: scan <= 2^22 points, <= 256 boxes,
 *            <= 64 masks, each bbox 0 <= l <= r <= img_w and 0 <= t <= b <= img_h after truncation.
 *   results  the arrays of the last run, box after box: points (sum n_pts x 3), depth (sum n_pts), rays
 *            (sum of n_rays > 0, x 3).  Any pointer may be NULL.
 * Beside a running keyframe: while the handle is alive, the solvers on its device leave DSPGN_FRAME_RESERVE_SMS SMs
 * free (dspgn_keyframe_submit), and the handle's own stream has the device's greatest priority, so its blocks are
 * dispatched ahead of a solver's queued kernels: a run does not wait for LocalMapping's keyframe.  A run allocates
 * nothing once its buffers are large enough; the first run with more scan points, boxes or masks than any before may
 * grow them (+25 % headroom), and freeing the old buffer waits for all work on the device, the keyframe included. */
typedef struct DspgnLidarFrame DspgnLidarFrame;
typedef struct {
  float k[9];                 /* K (3x3 row-major, float32 as the loader casts it) */
  float inv_k[9];             /* inv(K) as float32 */
  float t_cam_velo[16];       /* 4x4 row-major */
  int32_t img_h, img_w;       /* 1..4096 */
  int32_t num_lidar_max;      /* 1..4096 */
  int32_t min_mask_area;
  int32_t downsample_ratio;   /* int(configs.downsample_ratio), >= 1 */
  int32_t reserved_;
} DspgnLidarSpec;
typedef struct {
  float t_obj_velo[12];       /* rows 0..2 of inv(T_velo_obj) (float32 LAPACK on the host) */
  float trans[3];             /* box centre x, y, z (velodyne frame) */
  float size[3];              /* w, l, h */
  int32_t front;              /* T_cam_obj[2][3] > 0 as the caller computed T_cam_obj = T_cam_velo T_velo_obj */
} DspgnLidarBox;
typedef struct {
  int32_t n_pts;              /* surface points after subsampling */
  int32_t n_rays;             /* -1: no rays (None) */
  int32_t mask;               /* matched mask index, -1: none */
  int32_t n_selected;         /* points inside the box before subsampling */
} DspgnLidarBoxOut;
int dspgn_lidar_frame_create(const DspgnLidarSpec* spec, int device, DspgnLidarFrame** out);
void dspgn_lidar_frame_destroy(DspgnLidarFrame* f);
/* the handle enqueues on a non-blocking stream of its own (greatest priority); stream = a cudaStream_t replaces it
 * (NULL = legacy default; the caller's stream keeps the caller's priority) */
int dspgn_lidar_frame_set_stream(DspgnLidarFrame* f, void* cuda_stream);
/* scan: n_points x 4 float32 (x, y, z, reflectance); masks: n_masks x img_h x img_w bytes (numpy bool, nonzero =
 * inside); bboxes: n_masks x 4 int32 (l, t, r, b), the masks' boxes truncated like astype(int32) */
int dspgn_lidar_frame_run(DspgnLidarFrame* f, const float* scan, int n_points, const DspgnLidarBox* boxes, int n_boxes,
                          const uint8_t* masks, const int32_t* bboxes, int n_masks, DspgnLidarBoxOut* out);
int dspgn_lidar_frame_results(DspgnLidarFrame* f, float* points, float* depth, float* rays);

/* ---- A monocular (Redwood / Freiburg) keyframe's detection (mono_sequence.Frame.get_detections,
 * reconstruct/mono_sequence.py:75-114) and its keypoint test (Tracking::GetObjectDetectionsMono,
 * src/Tracking_util.cc:176-201), built on the device from the 2D masks and the keyframe's keypoints.  Its own handle,
 * like DspgnLidarFrame: Tracking is a different thread from LocalMapping's solver calls.
 *   mask      the first mask with the most set pixels (np.argmax of the areas); -1 when there are no masks.
 *   rays      the background grid of its bbox (truncated, expanded by 5 px, clamped; np.linspace(t, b, int(H/alpha))
 *             x np.linspace(l, r, int(W/alpha)), row-major) outside the mask, 200 of them at np.linspace(0, n-1, 200)
 *             ranks when more; undistorted as cv2.undistortPoints(pixels, K, (k1, k2, 0, 0, 0), P=K) (fp64, 5
 *             iterations, float32 result); rays = inv_k [u, v, 1] in float64, cast to float32.  Fewer than 2 such
 *             pixels is a frame the reference fails on (cv2 asserts on none, get_rays raises on one): n_rays = -1.
 *   features  the indices, ascending, of the keypoints whose pixel ((int)pt.y, (int)pt.x) is set in the mask eroded
 *             by getStructuringElement(MORPH_ELLIPSE, (2e+1)^2): every mask pixel of the ellipse around it that lies
 *             inside the image is set.  The image is not eroded: only the keypoints' footprints are read.
 * Every float step is rounded as numpy / OpenCV round it, so the arrays are bit-identical to the reference's.
 *   run      validates (DSPGN_E_ARG before anything is enqueued), stages the masks, bboxes and keypoints in pinned
 *            memory, one H2D copy, two kernels and one D2H copy on the handle's stream, then waits for that copy (the
 *            only host synchronisation) and writes the DspgnMonoOut.  Limits: <= 64 masks, each bbox 0 <= l <= r <=
 *            img_w and 0 <= t <= b <= img_h after truncation, <= 2^20 keypoints, each finite with -1 < x < img_w and
 *            -1 < y < img_h (its truncation inside the image).
 *   results  the arrays of the last run: background_rays (n_rays x 3, when n_rays > 0), feature_idx (n_feature).
 *            Either pointer may be NULL.
 * Beside a running keyframe: as DspgnLidarFrame (the SM reserve, the stream priority, and growth only on the first run
 * with more masks or keypoints than any before). */
typedef struct DspgnMonoFrame DspgnMonoFrame;
typedef struct {
  double k[9];                /* K_cam (3x3 row-major, float64 from the yaml's Camera.fx/fy/cx/cy) */
  double inv_k[9];            /* np.linalg.inv(K_cam), float64 */
  double k1, k2;              /* Camera.k1, Camera.k2 */
  int32_t img_h, img_w;       /* 1..4096 */
  int32_t downsample_ratio;   /* int(configs.downsample_ratio), >= 1 */
  int32_t mask_erosion;       /* Objects.maskErrosion, 0..63 */
} DspgnMonoSpec;
typedef struct {
  int32_t mask;               /* the largest mask's index, -1: no masks */
  int32_t n_nonsurface;       /* background pixels before subsampling */
  int32_t n_rays;             /* background rays, -1: none (no masks, or fewer than 2 pixels) */
  int32_t n_feature;          /* keypoints inside the eroded mask (the detection is good iff >= 20) */
} DspgnMonoOut;
int dspgn_mono_frame_create(const DspgnMonoSpec* spec, int device, DspgnMonoFrame** out);
void dspgn_mono_frame_destroy(DspgnMonoFrame* f);
/* as dspgn_lidar_frame_set_stream */
int dspgn_mono_frame_set_stream(DspgnMonoFrame* f, void* cuda_stream);
/* masks: n_masks x img_h x img_w bytes (numpy bool, nonzero = inside); bboxes: n_masks x 4 int32 (l, t, r, b), the
 * boxes truncated like astype(int32); keypoints: n_kp x 2 float32 (pt.x, pt.y of KeyFrame::mvKeys) */
int dspgn_mono_frame_run(DspgnMonoFrame* f, const uint8_t* masks, const int32_t* bboxes, int n_masks,
                         const float* keypoints, int n_kp, DspgnMonoOut* out);
int dspgn_mono_frame_results(DspgnMonoFrame* f, float* background_rays, int32_t* feature_idx);

/* Test hook for the wgmma operand paths: D[128][n_mma] = A[128][16*k_steps] * B[n_mma][16*k_steps]^T
 * (A through the register / shared-memory split-fp16 path, B through the pre-swizzled shared-memory images). Host buffers. */
int dspgn_tc_selftest(int device, int n_mma, int k_steps, const float* A, const float* B, float* D);

#ifdef __cplusplus
}
#endif
#endif /* DSPGN_H_ */
