// libdspgn.so host side: handles, weight packing, batch upload, launch sequencing.  C ABI in
// include/dspgn.h.  No torch, no exceptions across the boundary.
#include <cuda_runtime.h>
#include <cstdio>
#include <cstring>
#include <cmath>
#include <string>
#include <vector>
#include <memory>
#include <new>
#include <algorithm>
#include <atomic>
#include <mutex>
#include <thread>

#include <cub/device/device_scan.cuh>

#include "dspgn_common.cuh"
#include "dspgn_simt.cuh"
#include "dspgn_solve.cuh"
#include "dspgn_tc.cuh"
#include "dspgn_tc_wide.cuh"
#include "dspgn_simt_persistent.cuh"
#include "dspgn_mesh.cuh"
#include "dspgn_frame.cuh"
#include "dspgn_mono.cuh"

using namespace dspgn;

namespace {

constexpr int kEvCap = 1 << 18;     // events of the persistent kernel's debug log (env DSPGN_CLK)

thread_local std::string g_err;

int fail(int code, const std::string& msg) { g_err = msg; return code; }

#define CU(call)                                                                          \
  do {                                                                                    \
    cudaError_t e_ = (call);                                                              \
    if (e_ != cudaSuccess)                                                                \
      return fail(DSPGN_E_CUDA, std::string(#call) + ": " + cudaGetErrorString(e_));      \
  } while (0)

// A buffer that only grows, in device memory (DevBuf) or pinned host memory (HostBuf)
template <cudaError_t (*Alloc)(void**, size_t), cudaError_t (*Free)(void*)>
struct Buf {
  void* p = nullptr;
  size_t cap = 0;
  int reserve(size_t bytes) {
    if (bytes <= cap) return 0;
    if (p) Free(p);
    p = nullptr; cap = 0;
    size_t want = bytes + bytes / 4 + 256;
    if (Alloc(&p, want) != cudaSuccess) { cudaGetLastError(); return -1; }
    cap = want;
    return 0;
  }
  void release() { if (p) Free(p); p = nullptr; cap = 0; }
  template <class T> T* as() const { return reinterpret_cast<T*>(p); }
};

using DevBuf = Buf<cudaMalloc, cudaFree>;
using HostBuf = Buf<cudaMallocHost, cudaFreeHost>;   // pinned staging

}  // namespace

struct DspgnDecoder {
  int device = 0;
  bool has_ln = false;
  int hid = kHid;            // row stride of the SIMT weight images: kHidWide for a decoder with a layer wider than kHid
  DspgnDecoderSpec spec{};
  DecoderDev dev{};
  std::vector<void*> allocs;
  TcDecoderHost tc;
  // DSPGN_ENGINE_TC_WIDE images, built by the first solver that asks for that engine (tcw_pack_decoder).  Solvers
  // may be created from one decoder on several host threads: the build runs once, under the mutex, and a declined
  // shape is recorded so that it is not downloaded again.
  std::mutex tcw_mu;
  bool tcw_declined = false;
  TcDecoderHost tcw;
  TcPlan tcw_plan{};
};

struct DspgnSolver {
  int device = 0;
  int num_sms = 0;
  int engine = DSPGN_ENGINE_SIMT;
  int simt_hid = kHid;       // SIMT instantiation of the solver: its widest class's row stride
  DspgnConfig cfg{};
  cudaStream_t stream = nullptr;
  std::vector<DspgnDecoder*> classes;
  DevBuf d_decs;
  std::vector<void*> wide_allocs;  // kHidWide-stride weight images of the narrow classes of a wide solver
  // resident batch
  int n_obj = 0;
  int tot_pts = 0, tot_rays = 0, tot_fg = 0;
  long long tot_smp = 0;
  int max_rays = 0;
  std::vector<ObjMeta> h_meta;
  HostBuf h_stage;
  DevBuf d_stage;        // one contiguous upload: meta | T_init | code_init | pts | rays | depth
  ObjMeta* d_meta = nullptr; float* d_Tinit = nullptr; float* d_code = nullptr;
  float* d_pts = nullptr; float* d_rays = nullptr; float* d_depth = nullptr;
  DevBuf d_state, d_part_s, d_part_r, d_tbase, d_V, d_m, d_results, d_active;
  DevBuf d_sdf, d_bx, d_bs, d_br;
  DevBuf d_dbg;
  DevBuf d_q_flag, d_q_ctr, d_tiles_left, d_obj_iter;   // persistent-kernel work queue
  int* d_tbase_static = nullptr;   // [n_obj] first SDF tile (engine tile height) of each object (inside the staging block)
  int* d_tbase_r_static = nullptr; // [n_obj] first band-tile partial slot of each object (capacity: its ray-sample tiles + 1)
  // per-run object table (layout: run_table)
  DevBuf d_run;
  HostBuf h_run;                   // pinned staging of the table; rewritten only after ev_run_upload
  cudaEvent_t ev_run_upload = nullptr;
  bool run_upload_pending = false;
  bool run_table_valid = false;    // d_run holds h_run for the resident batch (a repeated run skips the copy)
  bool run_table_gated = false;    // ... and it is the table of a gated run (it has link and t_map)
  int total_tiles = 0;             // SDF tiles of the batch at the engine's tile height (tile_rows)
  int max_tiles = 0;               // largest tile count of one term of one object (queue items hold 19 bits)
  bool mega_enabled = true;
  bool compact_rays = true;        // persistent kernel, render term: forward-only tiles over the valid-sample hulls only (env DSPGN_COMPACT_RAYS=0: all n_rays x D samples)
  DevBuf d_ev, d_seg, d_ln, d_vpre;
  DevBuf d_masks;                  // k_gn_persistent, k_wide_wgmma: per-CTA ReLU mask scratch (kTcMaskLayers x kTcEpiThreads uint4 per SM)
  DevBuf d_tcw;                    // DSPGN_ENGINE_TC_WIDE: TcwDecDev of every class
  bool events_on = false;          // env DSPGN_CLK: the persistent kernel writes its event log (dspgn_debug_events)
  HostBuf h_results;
  // counters
  DspgnCounters ctr{};
  bool timing = false;
  std::vector<cudaEvent_t> ev;
  size_t ev_used = 0;
  std::vector<cudaEvent_t> ev_solve;
  size_t evs_used = 0;
  cudaEvent_t ev_run0 = nullptr, ev_run1 = nullptr;
  cudaStream_t stream2 = nullptr;    // fork: the ray-sample forward pass runs beside the SDF-row pass
  cudaEvent_t ev_fork = nullptr, ev_join = nullptr;
  cudaEvent_t ev_upload = nullptr;   // the pinned staging block may be rewritten only after its last H2D copy finished
  bool upload_pending = false;
  bool mega_ran = false;             // the last run used the persistent kernel: check its abort flag with the results
  bool band_rows_pending = false;    // the persistent kernel's band-row total has not been added to ctr yet
  int n_bad = 0;                     // resident objects rejected at upload (status BAD_INPUT, never evaluated)
  // multi-GPU result exchange (rank 0 owns the buffer, the others map it through CUDA IPC)
  struct Gather {
    bool active = false, owner = false;
    unsigned char* base = nullptr;   // [2][n_slots][88] floats | flags[world] | ack
    int n_slots = 0, world = 0, rank = 0;
    size_t off_flags = 0, off_ack = 0;
    DevBuf d_slot_of, d_local;       // d_local: int err | long long wait_ns
    HostBuf h_out;
    int bound_n = -1;
  } gather;
  // mesh calls (dspgn_mesh_batch): query points and scan workspace of one chunk, the grids of the whole call
  DevBuf d_grid_pts, d_mgrid, d_mws, d_mscan_tmp, d_mout;
  HostBuf h_mbase;
  int mesh_n = 0, mesh_dim = 0;      // objects / grid size of the last mesh call (0: none)
  std::vector<float> mesh_v;         // its meshes, object after object
  std::vector<int32_t> mesh_f;
  std::vector<int32_t> mesh_grid_of; // meshed keyframe call: grid of each object in d_mgrid (-1: none); empty: grid o is object o's
  DevBuf d_mesh_sel;                 // meshed keyframe call, per chunk: grid slot | pair partner of each resident slot
  HostBuf h_mesh_sel;                // ... its pinned staging (rewritten only after the chunk's results came back)
  // a submitted keyframe call (dspgn_keyframe_submit .. dspgn_keyframe_wait)
  struct Flight {
    bool active = false;
    bool mesh = false;               // a mesh spec was given
    bool mega = false;               // the run used the persistent kernel
    bool render = false;             // ... and the per-iteration schedule's woken slots run the render term
    bool device_wake = false;        // the per-iteration schedule's second round was enqueued for every gated slot
    int n_obj = 0, slots = 0, n = 0, dim = 0, n_cand = 0, gc = 0;
    long long cap_v = 0, cap_f = 0;  // mesh arena (vertices | faces)
    size_t o_ctr = 0, o_base = 0, o_arena = 0;   // h_flight: records | queue counters | mesh bases | arena
    std::vector<int> order;          // walk order of the objects
    std::vector<float> pose_scale;   // KfWalk::pose_scale
    std::vector<int32_t> link, grid_of;
    MeshGrid g{};
    uint8_t* mask = nullptr; int* vscan = nullptr; int* fscan = nullptr;   // the chunk's scans, kept for an overflow
  } flight;
  HostBuf h_flight;
  cudaEvent_t ev_flight = nullptr;
  double arena_v = 4.0, arena_f = 8.0;     // arena estimate: vertices / faces per object and per dim^2 (grows)
  long long arena_force_v = 0, arena_force_f = 0;   // dspgn_debug_mesh_arena
  long long host_syncs = 0;          // dspgn_debug_host_syncs
  int sm_force = 0;                  // dspgn_debug_sm_budget (0: the automatic budget, grid_sms)
  // cooperative stop (dspgn_keyframe_stop): a host-mapped word the kernels read, one generation per stoppable call
  uint32_t* h_stop = nullptr;        // pinned, mapped; the generation of the last call a stop was requested for
  uint32_t* d_stop = nullptr;        // its device address
  std::atomic<uint32_t> stop_live{0};   // generation of the call in flight (0: none); read by dspgn_keyframe_stop
  uint32_t stop_gen = 0;             // generation of the current / last call
  const volatile uint8_t* stop_flag = nullptr;   // dspgn_solver_set_stop_flag
  cudaEvent_t ev_poll = nullptr;     // the waits that poll stop_flag
  int stop_at_obj = -1, stop_at_iter = -1;       // dspgn_debug_stop_at, for the next stoppable call
  int call_stop_obj = -1, call_stop_iter = -1;   // ... taken by the call in flight (caller object index)
  // pose information (dspgn_pose_information) of the last call that returned records: the solve keeps the last
  // linearisation of each of the call's slots in d_lin (lin_floats(code_len) floats per slot, every chunk of the call)
  DevBuf d_lin;
  int lin_base = -1;                 // d_lin slot of the resident chunk's slot 0; -1: the runs keep no linearisation
  bool info_valid = false;           // info_items describes the last call (set when its records are complete)
  std::vector<InfoItem> info_items;  // per object of that call
  DevBuf d_info;                     // dspgn_pose_information: items | info | status
  HostBuf h_info;
};

namespace {

// ---- SM budget of the solver's grid-sized launches ----------------------------------------------------------------
// The persistent kernels fill a whole SM per CTA (registers and shared memory), so while one runs on every SM no block
// of another kernel can start anywhere.  A live frame handle (DspgnLidarFrame / DspgnMonoFrame) on the device means a
// Tracking thread may build a keyframe's detections while LocalMapping's keyframe runs: the grid-sized launches then
// leave kFrameReserveSms SMs to it.  Counted per device, read at every launch (the builder may be created after the
// solver).  DESIGN §5 has the measurement this value comes from.
constexpr int kFrameReserveSms = DSPGN_FRAME_RESERVE_SMS;
constexpr int kMaxDevices = 64;
std::atomic<int> g_live_frames[kMaxDevices];

void count_frame(int device, int delta) {
  if (device >= 0 && device < kMaxDevices) g_live_frames[device].fetch_add(delta, std::memory_order_relaxed);
}

// rows per tile of the solver's decoder engine (the per-tile partial sums of a term: one slot per tile)
int tile_rows(const DspgnSolver* s) {
  if (s->engine == DSPGN_ENGINE_TC_WIDE) return kTcwRows;
  return (s->engine == DSPGN_ENGINE_TC) ? kTcRows : simt_rows(s->simt_hid);
}

// the SIMT engine's LayerNorm scratch of one grid-sized launch: [CTA][layer][H][rows] (TermArgs.ln_scratch)
size_t ln_half_floats(const DspgnSolver* s) {
  return (size_t)s->num_sms * DSPGN_MAX_LINEAR * s->simt_hid * simt_rows(s->simt_hid);
}

// CTAs of the next grid-sized launch (k_gn_persistent*, k_decoder_tc, k_decoder_simt): at most this many
int grid_sms(const DspgnSolver* s) {
  if (s->sm_force > 0) return s->sm_force;
  const bool frames = s->device < kMaxDevices && g_live_frames[s->device].load(std::memory_order_relaxed) > 0;
  return frames ? std::max(s->num_sms - kFrameReserveSms, 1) : s->num_sms;
}

// ---- cooperative stop (dspgn_keyframe_stop) ------------------------------------------------------------------------
// A stop of the call in flight: the word takes the call's generation, never an older generation over a newer one (a
// stop that races with the end of its call cannot cancel the next call's).
void request_stop(DspgnSolver* s) {
  const uint32_t g = s->stop_live.load(std::memory_order_acquire);
  if (g == 0) return;
  uint32_t cur = __atomic_load_n(s->h_stop, __ATOMIC_RELAXED);
  while (cur < g && !__atomic_compare_exchange_n(s->h_stop, &cur, g, true, __ATOMIC_RELEASE, __ATOMIC_RELAXED)) {}
}

void stop_end(DspgnSolver* s) {
  s->stop_live.store(0, std::memory_order_release);
  s->call_stop_obj = s->call_stop_iter = -1;
}

// The stoppable calls (dspgn_reconstruct_batch, the keyframe calls) hold one for their duration: a generation of their
// own, live until the call returns; a submitted call keeps it (keep = true) until its wait.  The call takes the test
// hook of dspgn_debug_stop_at.
struct StopScope {
  DspgnSolver* s;
  bool keep = false;
  explicit StopScope(DspgnSolver* s_) : s(s_) {
    s->stop_gen = s->stop_gen + 1;
    if (s->stop_gen == 0) {            // 2^32 calls: the word may hold a large old generation; no call is in flight
      __atomic_store_n(s->h_stop, 0u, __ATOMIC_RELAXED);
      s->stop_gen = 1;
    }
    s->call_stop_obj = s->stop_at_obj; s->call_stop_iter = s->stop_at_iter;
    s->stop_at_obj = s->stop_at_iter = -1;
    s->stop_live.store(s->stop_gen, std::memory_order_release);
  }
  ~StopScope() { if (!keep) stop_end(s); }
};

// The wait of a solver with a registered stop flag: the event and the flag polled in turn, yielding the core between
// polls -- a spin like the one a blocking synchronisation does under the runtime's default scheduling.  A timed sleep
// overshoots by the kernel's timer slack and, on a busy host, by milliseconds (DESIGN §5).
cudaError_t poll_event(DspgnSolver* s, cudaEvent_t e) {
  bool raised = false;
  for (;;) {
    const cudaError_t q = cudaEventQuery(e);
    if (q != cudaErrorNotReady) return q;
    if (!raised && *s->stop_flag != 0) { request_stop(s); raised = true; }
    std::this_thread::yield();
  }
}

// Every wait of the calling thread on the device goes through these (dspgn_debug_host_syncs counts them).
cudaError_t sync_stream(DspgnSolver* s) {
  ++s->host_syncs;
  if (s->stop_flag) {
    const cudaError_t e = cudaEventRecord(s->ev_poll, s->stream);
    return e != cudaSuccess ? e : poll_event(s, s->ev_poll);
  }
  return cudaStreamSynchronize(s->stream);
}

// Before a buffer the stream's earlier work may still read is freed or rewritten: waits only if that work is unfinished.
cudaError_t settle_stream(DspgnSolver* s) {
  const cudaError_t q = cudaStreamQuery(s->stream);
  if (q != cudaErrorNotReady) return q;
  return sync_stream(s);
}

cudaError_t settle_event(DspgnSolver* s, cudaEvent_t e) {
  const cudaError_t q = cudaEventQuery(e);
  if (q != cudaErrorNotReady) return q;
  ++s->host_syncs;
  return s->stop_flag ? poll_event(s, e) : cudaEventSynchronize(e);
}

// ---- a run's counters and timing (dspgn_counters) ------------------------------------------------------------------
// Every call that enqueues device work of its own (the runs, dspgn_decode_sdf, the mesh calls, the debug system hook)
// brackets it with run_begin .. run_end: the counters, the timed-launch event pools and ev_run0 / ev_run1 then describe
// that call.
int run_begin(DspgnSolver* s) {
  s->info_valid = false;             // the pose information belongs to the last call, and this is a new one
  s->ctr = DspgnCounters{};
  s->band_rows_pending = false;
  s->ev_used = 0;
  s->evs_used = 0;
  CU(cudaEventRecord(s->ev_run0, s->stream));
  return 0;
}

int run_end(DspgnSolver* s) {
  CU(cudaEventRecord(s->ev_run1, s->stream));
  return 0;
}

// The last run's device times, once its events have completed: decoder_ms and solve_ms from the event pairs of the
// timed launches (dspgn_enable_timing), total_ms from ev_run0 to ev_run1.
void read_timings(DspgnSolver* s) {
  float tot = 0.f;
  if (cudaEventElapsedTime(&tot, s->ev_run0, s->ev_run1) != cudaSuccess) { cudaGetLastError(); return; }
  s->ctr.total_ms = tot;
  auto pairs = [](const std::vector<cudaEvent_t>& ev, size_t used) {
    float sum = 0.f;
    for (size_t i = 0; i + 1 < used; i += 2) { float ms = 0.f; cudaEventElapsedTime(&ms, ev[i], ev[i + 1]); sum += ms; }
    return sum;
  };
  s->ctr.decoder_ms = pairs(s->ev, s->ev_used);
  s->ctr.solve_ms = pairs(s->ev_solve, s->evs_used);
}

#define BUSY(s)                                                                                              \
  do {                                                                                                       \
    if ((s) && (s)->flight.active)                                                                           \
      return fail(DSPGN_E_BUSY, "the solver has a submitted keyframe call that has not been collected (dspgn_keyframe_wait)"); \
  } while (0)

// what is concatenated at the input of layer k (latent_in_layer is shorthand for one kind-1 layer)
int cat_kind_of(const DspgnDecoderSpec& s, int k) {
  if (s.cat_kind[k] != 0) return s.cat_kind[k];
  return (k == s.latent_in_layer) ? 1 : 0;
}

int check_spec(const DspgnDecoderSpec& s) {
  if (s.num_linear < 3 || s.num_linear > 9) return fail(DSPGN_E_ARG, "num_linear must be in [3,9]");
  if (s.latent_size < 1 || s.latent_size > DSPGN_MAX_CODE) return fail(DSPGN_E_ARG, "latent_size must be <= 64");
  const int in0 = s.latent_size + 3;
  if (s.in_dim[0] != in0) return fail(DSPGN_E_ARG, "in_dim[0] must equal latent_size+3");
  if (s.out_dim[s.num_linear - 1] != 1) return fail(DSPGN_E_ARG, "last layer must have one output");
  if (s.latent_in_layer != -1 && (s.latent_in_layer < 1 || s.latent_in_layer > s.num_linear - 1))
    return fail(DSPGN_E_ARG, "latent_in_layer must be a layer index >= 1 or -1");
  for (int k = 0; k < s.num_linear; ++k) {
    if (s.in_dim[k] < 1 || s.in_dim[k] > kHidWide || s.out_dim[k] < 1 || s.out_dim[k] > kHidWide)
      return fail(DSPGN_E_ARG, "layer widths must be in [1,512]");
    const int ck = cat_kind_of(s, k);
    if (ck < 0 || ck > 2 || (k == 0 && ck != 0)) return fail(DSPGN_E_ARG, "bad cat_kind");
    if (s.layer_norm[k] != 0 && k == s.num_linear - 1) return fail(DSPGN_E_ARG, "the last layer cannot be normalised");
    if (k > 0) {
      const int expect = s.out_dim[k - 1] + (ck == 1 ? in0 : (ck == 2 ? 3 : 0));
      if (s.in_dim[k] != expect) return fail(DSPGN_E_ARG, "layer in_dim inconsistent with previous out_dim/latent_in");
    }
  }
  return 0;
}

int upload_vec(DspgnDecoder* d, const std::vector<float>& h, const float** out) {
  void* p = nullptr;
  CU(cudaMalloc(&p, h.size() * sizeof(float)));
  d->allocs.push_back(p);
  CU(cudaMemcpy(p, h.data(), h.size() * sizeof(float), cudaMemcpyHostToDevice));
  *out = reinterpret_cast<const float*>(p);
  return 0;
}

// The device of a new decoder or frame handle: present, an sm_90 part, and made current
int check_device(int device) {
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) { cudaGetLastError(); return fail(DSPGN_E_NOGPU, "no CUDA device"); }
  if (device < 0 || device >= ndev) return fail(DSPGN_E_ARG, "bad device index");
  CU(cudaSetDevice(device));
  cudaDeviceProp prop;
  CU(cudaGetDeviceProperties(&prop, device));
  if (prop.major != 9 || prop.minor != 0) return fail(DSPGN_E_NOGPU, "libdspgn is built for sm_90a (H100) only; found sm_" + std::to_string(prop.major) + std::to_string(prop.minor));
  return 0;
}

}  // namespace

extern "C" {

const char* dspgn_last_error(void) { return g_err.c_str(); }
int dspgn_version(void) { return 100; }

int dspgn_decoder_create(const DspgnDecoderSpec* spec, const float* const* W, const float* const* b,
                         int device, DspgnDecoder** out) {
  return dspgn_decoder_create_ex(spec, W, b, nullptr, nullptr, device, out);
}

int dspgn_decoder_create_ex(const DspgnDecoderSpec* spec, const float* const* W, const float* const* b,
                            const float* const* ln_gamma, const float* const* ln_beta, int device, DspgnDecoder** out) {
  if (!spec || !W || !b || !out) return fail(DSPGN_E_ARG, "null argument");
  for (int k = 0; k < spec->num_linear && k < DSPGN_MAX_LINEAR; ++k)
    if (spec->layer_norm[k] && (!ln_gamma || !ln_beta || !ln_gamma[k] || !ln_beta[k])) return fail(DSPGN_E_ARG, "LayerNorm parameters missing");
  if (int rc = check_spec(*spec)) return rc;
  if (int rc = check_device(device)) return rc;
  DspgnDecoder* d = new (std::nothrow) DspgnDecoder();
  if (!d) return fail(DSPGN_E_ALLOC, "oom");
  d->device = device;
  d->spec = *spec;
  DecoderDev& dv = d->dev;
  dv.L = spec->latent_size; dv.n_lin = spec->num_linear; dv.in0 = spec->latent_size + 3;
  const int nl = spec->num_linear;
  // variants: the plain shape (at most one latent_in layer among the hidden layers, nothing else) runs on both engines
  int n_cat1 = 0, cat1_layer = -1;
  bool generic = spec->use_tanh != 0;
  for (int k = 0; k < nl; ++k) {
    dv.cat_kind[k] = cat_kind_of(*spec, k);
    if (dv.cat_kind[k] == 1) { ++n_cat1; cat1_layer = k; }
    if (dv.cat_kind[k] == 2 || spec->layer_norm[k]) generic = true;
  }
  if (n_cat1 > 1 || (n_cat1 == 1 && cat1_layer > nl - 2)) generic = true;
  dv.latent_in = (n_cat1 == 1) ? cat1_layer : -1;
  dv.use_tanh = spec->use_tanh != 0; dv.generic = generic ? 1 : 0;
  d->has_ln = false;
  for (int k = 0; k < nl; ++k)
    if (spec->in_dim[k] > kHid || spec->out_dim[k] > kHid) d->hid = kHidWide;
  const int H = d->hid;
  int rc = 0;
  for (int k = 0; k < nl && rc == 0; ++k) {
    const int nin = spec->in_dim[k], nout = spec->out_dim[k];
    dv.in_dim[k] = nin; dv.out_dim[k] = nout;
    const int in_pad = (nin + kKC - 1) / kKC * kKC, out_pad = (nout + kKC - 1) / kKC * kKC;
    std::vector<float> wf((size_t)in_pad * H, 0.f), wb((size_t)out_pad * H, 0.f), bb(H, 0.f);
    for (int j = 0; j < nout; ++j) {
      for (int i = 0; i < nin; ++i) {
        const float w = W[k][(size_t)j * nin + i];
        wf[(size_t)i * H + j] = w;
        wb[(size_t)j * H + i] = w;
      }
      bb[j] = b[k][j];
    }
    rc = upload_vec(d, wf, &dv.Wf[k]);
    if (!rc) rc = upload_vec(d, wb, &dv.Wb[k]);
    if (!rc) rc = upload_vec(d, bb, &dv.bias[k]);
    if (!rc && k == nl - 1) {
      std::vector<float> wl(H, 0.f);
      for (int i = 0; i < nin; ++i) wl[i] = W[k][i];
      rc = upload_vec(d, wl, &dv.w_last);
    }
    if (!rc && spec->layer_norm[k]) {
      std::vector<float> g(H, 0.f), be(H, 0.f);
      for (int j = 0; j < nout; ++j) { g[j] = ln_gamma[k][j]; be[j] = ln_beta[k][j]; }
      rc = upload_vec(d, g, &dv.ln_gamma[k]);
      if (!rc) rc = upload_vec(d, be, &dv.ln_beta[k]);
      d->has_ln = true;
    }
  }
  if (!rc && !generic) rc = tc_pack_decoder(*spec, W, b, d->tc, &dv, g_err);     // the tensor-core engine covers the plain shape
  if (rc) { dspgn_decoder_destroy(d); return rc; }
  *out = d;
  return 0;
}

void dspgn_decoder_destroy(DspgnDecoder* d) {
  if (!d) return;
  cudaSetDevice(d->device);
  for (void* p : d->allocs) cudaFree(p);
  tc_free_decoder(d->tc);
  tc_free_decoder(d->tcw);
  delete d;
}

int dspgn_solver_create(const DspgnConfig* cfg, DspgnDecoder* const* classes, int n_classes, int device,
                        DspgnSolver** out) {
  if (!cfg || !classes || !out) return fail(DSPGN_E_ARG, "null argument");
  if (n_classes < 1 || n_classes > DSPGN_MAX_CLASSES) return fail(DSPGN_E_ARG, "n_classes must be in [1,4]");
  if (cfg->num_depth_samples < 2 || cfg->num_depth_samples > kMaxDepthSamples)
    return fail(DSPGN_E_ARG, "num_depth_samples must be in [2,256]");
  if (cfg->num_iterations < 1) return fail(DSPGN_E_ARG, "num_iterations must be >= 1");
  for (int c = 0; c < n_classes; ++c) {
    if (!classes[c] || classes[c]->device != device) return fail(DSPGN_E_ARG, "decoder/device mismatch");
    if (cfg->code_len < 1 || cfg->code_len > classes[c]->spec.latent_size) return fail(DSPGN_E_ARG, "code_len exceeds decoder latent_size");
    // code_len < latent_size: the trailing latent entries stay zero and are not optimised (optimizer.py:97-100
    // slices code[:code_len]; the reference itself needs code_len == latent size for its decoder input)
  }
  CU(cudaSetDevice(device));
  // every failure below releases the half-built solver (events, streams, device buffers)
  std::unique_ptr<DspgnSolver, decltype(&dspgn_solver_destroy)> owner(new (std::nothrow) DspgnSolver(), dspgn_solver_destroy);
  DspgnSolver* s = owner.get();
  if (!s) return fail(DSPGN_E_ALLOC, "oom");
  s->device = device;
  s->cfg = *cfg;
  cudaDeviceProp prop;
  CU(cudaGetDeviceProperties(&prop, device));
  s->num_sms = prop.multiProcessorCount;
  for (int c = 0; c < n_classes; ++c) s->classes.push_back(classes[c]);
  std::vector<DecoderDev> decs;
  for (auto* d : s->classes) s->simt_hid = std::max(s->simt_hid, d->hid);
  for (auto* d : s->classes) {
    decs.push_back(d->dev);
    if (d->hid == s->simt_hid) continue;
    // a narrow class of a wide solver runs in the wide instantiation: its matrices again at the wider row stride
    DecoderDev& dv = decs.back();
    for (int k = 0; k < dv.n_lin; ++k)
      for (const float** m : {&dv.Wf[k], &dv.Wb[k]}) {
        const size_t rows = (size_t)((m == &dv.Wf[k] ? dv.in_dim[k] : dv.out_dim[k]) + kKC - 1) / kKC * kKC;
        void* p = nullptr;
        CU(cudaMalloc(&p, rows * s->simt_hid * sizeof(float)));
        s->wide_allocs.push_back(p);
        CU(cudaMemset(p, 0, rows * s->simt_hid * sizeof(float)));
        CU(cudaMemcpy2D(p, s->simt_hid * sizeof(float), *m, d->hid * sizeof(float), d->hid * sizeof(float), rows,
                        cudaMemcpyDeviceToDevice));
        *m = static_cast<const float*>(p);
      }
  }
  if (s->d_decs.reserve(decs.size() * sizeof(DecoderDev))) return fail(DSPGN_E_ALLOC, "cudaMalloc");
  CU(cudaMemcpy(s->d_decs.p, decs.data(), decs.size() * sizeof(DecoderDev), cudaMemcpyHostToDevice));
  bool tc_ok = true;
  for (auto* d : s->classes) tc_ok = tc_ok && d->tc.ok;
  int eng = cfg->engine;
  if (eng == DSPGN_ENGINE_AUTO) {
    const char* e = getenv("DSPGN_ENGINE");
    if (e && !strcmp(e, "simt")) eng = DSPGN_ENGINE_SIMT;
    else if (e && !strcmp(e, "tc")) eng = DSPGN_ENGINE_TC;
    else eng = (tc_ok && tc_engine_default()) ? DSPGN_ENGINE_TC : DSPGN_ENGINE_SIMT;
  }
  if (eng == DSPGN_ENGINE_TC && !tc_ok) return fail(DSPGN_E_ARG, "tensor-core engine unavailable for this decoder shape");
  if (eng == DSPGN_ENGINE_TC_WIDE) {
    std::vector<TcwDecDev> wd;
    for (auto* d : s->classes) {
      std::lock_guard<std::mutex> lock(d->tcw_mu);
      if (!d->tcw.ok && !d->tcw_declined) {
        if (int rc = tcw_pack_decoder(d->dev, d->hid, d->tcw, d->tcw_plan, g_err)) return rc;
        d->tcw_declined = !d->tcw.ok;
      }
      if (d->tcw_declined)
        return fail(DSPGN_E_ARG, "wide tensor-core engine (DSPGN_ENGINE_TC_WIDE) unavailable for this decoder shape: plain "
                                 "decoders only (no LayerNorm, xyz_in_all, use_tanh or second latent_in layer)");
      wd.push_back(TcwDecDev{reinterpret_cast<const unsigned char*>(d->tcw.blob), d->tcw_plan});
    }
    if (s->d_tcw.reserve(wd.size() * sizeof(TcwDecDev))) return fail(DSPGN_E_ALLOC, "cudaMalloc");
    CU(cudaMemcpy(s->d_tcw.p, wd.data(), wd.size() * sizeof(TcwDecDev), cudaMemcpyHostToDevice));
    if (int rc = tcw_setup_kernel(g_err)) return rc;
  }
  s->engine = eng;
  if (s->simt_hid == kHid)
    CU(cudaFuncSetAttribute(k_decoder_simt<kHid>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(SimtSmem<kHid>)));
  else
    CU(cudaFuncSetAttribute(k_decoder_simt<kHidWide>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(SimtSmem<kHidWide>)));
  if (int rc = simt_setup_kernels(s->simt_hid, g_err)) return rc;
  for (auto* d : s->classes)
    if (d->has_ln) {      // LayerNorm decoders: per-CTA scratch for the normalised activations (forward -> backward),
                          // one half for the ray-sample pass, which may run beside the SDF-row pass (launch_terms)
      if (s->d_ln.reserve(4 * 2 * ln_half_floats(s))) return fail(DSPGN_E_ALLOC, "cudaMalloc");
      break;
    }
  static_assert(kTcwMaskLayers <= kTcMaskLayers, "d_masks holds kTcMaskLayers layers per CTA, k_wide_wgmma strides by kTcwMaskLayers");
  if ((eng == DSPGN_ENGINE_TC || eng == DSPGN_ENGINE_TC_WIDE) &&
      s->d_masks.reserve(sizeof(uint4) * (size_t)s->num_sms * kTcMaskLayers * kTcEpiThreads)) return fail(DSPGN_E_ALLOC, "cudaMalloc");
  if (int rc = tc_setup_kernels(g_err)) return rc;
  if (const char* m = getenv("DSPGN_MEGA")) s->mega_enabled = (m[0] != '0');
  if (const char* m = getenv("DSPGN_COMPACT_RAYS")) s->compact_rays = (m[0] != '0');   // A/B switch of the valid-sample hulls
  if (cfg->schedule == DSPGN_SCHED_LAUNCHES) s->mega_enabled = false;
  else if (cfg->schedule == DSPGN_SCHED_PERSISTENT) s->mega_enabled = true;
  else if (cfg->schedule != DSPGN_SCHED_AUTO) return fail(DSPGN_E_ARG, "bad schedule");
  s->events_on = getenv("DSPGN_CLK") != nullptr;
  CU(cudaEventCreateWithFlags(&s->ev_upload, cudaEventDisableTiming));
  CU(cudaEventCreateWithFlags(&s->ev_run_upload, cudaEventDisableTiming));
  CU(cudaStreamCreateWithFlags(&s->stream2, cudaStreamNonBlocking));
  CU(cudaEventCreateWithFlags(&s->ev_fork, cudaEventDisableTiming));
  CU(cudaEventCreateWithFlags(&s->ev_join, cudaEventDisableTiming));
  CU(cudaEventCreate(&s->ev_run0));
  CU(cudaEventCreate(&s->ev_run1));
  CU(cudaEventCreateWithFlags(&s->ev_poll, cudaEventDisableTiming));
  CU(cudaHostAlloc(reinterpret_cast<void**>(&s->h_stop), sizeof(uint32_t), cudaHostAllocMapped));
  *s->h_stop = 0;
  CU(cudaHostGetDevicePointer(reinterpret_cast<void**>(&s->d_stop), s->h_stop, 0));
  *out = owner.release();
  return 0;
}

void dspgn_solver_destroy(DspgnSolver* s) {
  if (!s) return;
  cudaSetDevice(s->device);
  cudaDeviceSynchronize();                 // also the work of a submitted call that was never collected
  s->flight.active = false;
  dspgn_gather_close(s);
  for (DevBuf* b : {&s->d_decs, &s->d_stage, &s->d_state, &s->d_part_s, &s->d_part_r, &s->d_tbase, &s->d_V, &s->d_m, &s->d_results, &s->d_active,
                    &s->d_sdf, &s->d_bx, &s->d_bs, &s->d_br, &s->d_dbg, &s->d_q_flag, &s->d_q_ctr,
                    &s->d_tiles_left, &s->d_obj_iter, &s->d_ev, &s->d_seg, &s->d_ln, &s->d_vpre, &s->d_masks, &s->d_tcw, &s->d_run,
                    &s->d_grid_pts, &s->d_mgrid, &s->d_mws, &s->d_mscan_tmp, &s->d_mout, &s->d_mesh_sel, &s->d_lin, &s->d_info}) b->release();
  for (void* p : s->wide_allocs) cudaFree(p);
  s->h_stage.release();
  s->h_mbase.release();
  s->h_results.release();
  s->h_run.release();
  s->h_mesh_sel.release();
  s->h_flight.release();
  s->h_info.release();
  if (s->ev_flight) cudaEventDestroy(s->ev_flight);
  for (auto e : s->ev) cudaEventDestroy(e);
  for (auto e : s->ev_solve) cudaEventDestroy(e);
  if (s->ev_upload) cudaEventDestroy(s->ev_upload);
  if (s->ev_run_upload) cudaEventDestroy(s->ev_run_upload);
  if (s->ev_fork) cudaEventDestroy(s->ev_fork);
  if (s->ev_join) cudaEventDestroy(s->ev_join);
  if (s->stream2) cudaStreamDestroy(s->stream2);
  if (s->ev_run0) cudaEventDestroy(s->ev_run0);
  if (s->ev_run1) cudaEventDestroy(s->ev_run1);
  if (s->ev_poll) cudaEventDestroy(s->ev_poll);
  if (s->h_stop) cudaFreeHost(s->h_stop);
  delete s;
}

int dspgn_solver_set_stream(DspgnSolver* s, void* cuda_stream) {
  if (!s) return fail(DSPGN_E_ARG, "null solver");
  BUSY(s);
  s->stream = reinterpret_cast<cudaStream_t>(cuda_stream);
  return 0;
}

int dspgn_solver_engine(const DspgnSolver* s) { return s ? s->engine : DSPGN_E_ARG; }

int dspgn_solver_sync(DspgnSolver* s) {
  if (!s) return fail(DSPGN_E_ARG, "null solver");
  CU(cudaSetDevice(s->device));
  CU(sync_stream(s));
  return 0;
}

int dspgn_enable_timing(DspgnSolver* s, int on) {
  if (!s) return fail(DSPGN_E_ARG, "null solver");
  BUSY(s);
  s->timing = on != 0;
  return 0;
}

int dspgn_counters(DspgnSolver* s, DspgnCounters* out) {
  if (!s || !out) return fail(DSPGN_E_ARG, "null argument");
  BUSY(s);
  read_timings(s);
  *out = s->ctr;
  return 0;
}

// ---------------------------------------------------------------------------------------------
namespace {

// The SDF tiles and ray-sample tiles of one object at `rows` rows per tile.  k_init counts an object's tiles by the
// same rule on the device, at InitArgs.tile_rows (ntS, ntF_cap): the two must agree, for k_init seeds the iteration-0
// queue slots that plan_run reserves.
struct ObjTiles { long long sdf, smp; };
ObjTiles obj_tiles(const ObjMeta& M, int D, int rows) {
  return ObjTiles{(M.n_pts + rows - 1) / rows, ((long long)M.n_rays * D + rows - 1) / rows};
}

// decode_only: forward-only use (dspgn_decode_sdf) -- no J^T J partials, no band buffers.
// grid_dim > 0 (mesh calls, decode_only): every object's points are the dim^3 query grid, written on the device into a
// block of their own (in[o].pts is ignored, in[o].n_pts must be dim^3).
int upload_batch_impl(DspgnSolver* s, int n_obj, const DspgnObjectIn* in, bool decode_only, int grid_dim = 0) {
  if (!s || !in) return fail(DSPGN_E_ARG, "null argument");
  if (n_obj < 1 || n_obj > kMaxObjScan) return fail(DSPGN_E_ARG, "n_obj must be in [1,1024] per resident batch");
  CU(cudaSetDevice(s->device));
  const int D = s->cfg.num_depth_samples;
  s->h_meta.assign(n_obj, ObjMeta{});
  long long tp = 0, tr = 0, tf = 0, ts = 0;
  int max_rays = 0, n_bad = 0, any_build = 0;
  for (int o = 0; o < n_obj; ++o) {
    const DspgnObjectIn& I = in[o];
    // misuse of the API fails the call; an unusable DETECTION only fails that object (status BAD_INPUT ->
    // is_good=False), like the reference's soft exits (optimizer.py:130-150): one bad object must neither abort
    // its batch neighbours nor raise inside the embedded interpreter
    if (!I.t_cam_obj) return fail(DSPGN_E_ARG, "object without a pose");
    if (I.class_id < 0 || I.class_id >= (int)s->classes.size()) return fail(DSPGN_E_ARG, "bad class_id");
    const bool bad = I.n_pts < 1 || (!I.pts && grid_dim == 0) || I.n_rays < 0 || I.n_depth < 0 || I.n_depth > I.n_rays ||
                     I.n_rays > kScanMaxRays || (I.n_rays > 0 && I.n_depth > 0 && !I.depth) || (I.pixels && !I.inv_k);
    const float* ray_src = I.pixels ? I.pixels : I.rays;
    ObjMeta& M = s->h_meta[o];
    M.bad = bad ? 1 : 0;
    M.pts_off = (int)tp; M.n_pts = bad ? 0 : I.n_pts;
    M.ray_off = (int)tr; M.n_rays = (!bad && ray_src) ? I.n_rays : 0; M.n_fg = (!bad && ray_src) ? I.n_depth : 0;
    M.build = bad ? 0 : ((I.pixels ? 1 : 0) | (I.t_cam_world ? 2 : 0));
    any_build |= M.build;
    M.fg_off = (int)tf; M.smp_off = (int)ts;
    M.class_id = I.class_id; M.scale = I.scale; M.has_code = I.code != nullptr;
    tp += M.n_pts; tr += M.n_rays; tf += M.n_fg; ts += (long long)M.n_rays * D;
    if (M.n_rays > max_rays) max_rays = M.n_rays;
    n_bad += M.bad;
  }
  s->n_bad = n_bad;
  if (tp > (1 << 28) || ts > (1LL << 30)) return fail(DSPGN_E_ARG, "batch too large");
  // one staging block: meta | T_init | code | pts | rays | depth
  auto al = [](size_t x) { return (x + 255) / 256 * 256; };
  const size_t o_meta = 0, o_T = al(o_meta + sizeof(ObjMeta) * n_obj), o_code = al(o_T + 64 * n_obj),
               o_pts = al(o_code + 4 * kMaxCode * (size_t)n_obj), o_rays = al(o_pts + (grid_dim ? 0 : 12 * (size_t)tp)),
               o_depth = al(o_rays + 12 * (size_t)tr), o_tb = al(o_depth + 4 * (size_t)tf),
               o_aux = al(o_tb + 2 * 4 * (size_t)n_obj),
               total = al(o_aux + (any_build ? 4 * (size_t)kAuxFloats * n_obj : 0));
  if (s->upload_pending) { CU(settle_event(s, s->ev_upload)); s->upload_pending = false; }
  if (s->d_stage.cap < total) CU(settle_stream(s));      // kernels of an earlier batch may still read the old block
  if (s->h_stage.reserve(total) || s->d_stage.reserve(total)) return fail(DSPGN_E_ALLOC, "staging allocation failed");
  unsigned char* hb = s->h_stage.as<unsigned char>();
  memcpy(hb + o_meta, s->h_meta.data(), sizeof(ObjMeta) * n_obj);
  float* hT = reinterpret_cast<float*>(hb + o_T);
  float* hC = reinterpret_cast<float*>(hb + o_code);
  float* hP = reinterpret_cast<float*>(hb + o_pts);
  float* hR = reinterpret_cast<float*>(hb + o_rays);
  float* hD = reinterpret_cast<float*>(hb + o_depth);
  int* hTB = reinterpret_cast<int*>(hb + o_tb);
  {
    int acc = 0, mx = 0;
    long long accr = 0;
    int* hTBr = hTB + n_obj;
    const int rows = tile_rows(s);
    for (int o = 0; o < n_obj; ++o) {
      const ObjTiles t = obj_tiles(s->h_meta[o], D, rows);
      const int nt = (int)t.sdf, ntf = (int)t.smp;
      hTB[o] = acc; hTBr[o] = (int)(accr + o);
      acc += nt; accr += ntf;
      if (nt > mx) mx = nt;
      if (ntf > mx) mx = ntf;
    }
    s->total_tiles = acc; s->max_tiles = mx;
  }
  for (int o = 0; o < n_obj; ++o) {
    const DspgnObjectIn& I = in[o];
    const ObjMeta& M = s->h_meta[o];
    for (int r = 0; r < 4; ++r)
      for (int c = 0; c < 4; ++c) hT[o * 16 + r * 4 + c] = I.t_cam_obj[(size_t)r * I.t_rs + (size_t)c * I.t_cs];
    for (int i = 0; i < kMaxCode; ++i) hC[o * kMaxCode + i] = (I.code && i < s->cfg.code_len) ? I.code[i] : 0.f;
    float* p = hP + 3 * (size_t)M.pts_off;
    const int n_host_pts = grid_dim ? 0 : M.n_pts;
    if (n_host_pts > 0 && I.pts_cs == 1 && I.pts_rs == 3) memcpy(p, I.pts, 12 * (size_t)M.n_pts);
    else for (int r = 0; r < n_host_pts; ++r)
      for (int c = 0; c < 3; ++c) p[3 * (size_t)r + c] = I.pts[(size_t)r * I.pts_rs + (size_t)c * I.pts_cs];
    float* q = hR + 3 * (size_t)M.ray_off;
    if (M.build & 1) {                      // pixel coordinates: the device turns (u, v, 1) into inv_k [u, v, 1]
      for (int r = 0; r < M.n_rays; ++r) {
        q[3 * (size_t)r] = I.pixels[(size_t)r * I.pix_rs]; q[3 * (size_t)r + 1] = I.pixels[(size_t)r * I.pix_rs + I.pix_cs];
        q[3 * (size_t)r + 2] = 1.f;
      }
    } else
    for (int r = 0; r < M.n_rays; ++r)
      for (int c = 0; c < 3; ++c) q[3 * (size_t)r + c] = I.rays[(size_t)r * I.rays_rs + (size_t)c * I.rays_cs];
    if (any_build) {
      float* ax = reinterpret_cast<float*>(hb + o_aux) + (size_t)o * kAuxFloats;
      for (int i = 0; i < kAuxFloats; ++i) ax[i] = 0.f;
      if (M.build & 1) for (int i = 0; i < 9; ++i) ax[i] = I.inv_k[i];
      if (M.build & 2) for (int i = 0; i < 12; ++i) ax[9 + i] = I.t_cam_world[i];
    }
    if (M.n_fg) memcpy(hD + M.fg_off, I.depth, 4 * (size_t)M.n_fg);
  }
  CU(cudaMemcpyAsync(s->d_stage.p, hb, total, cudaMemcpyHostToDevice, s->stream));
  CU(cudaEventRecord(s->ev_upload, s->stream));
  s->upload_pending = true;
  unsigned char* db = s->d_stage.as<unsigned char>();
  if (any_build) {                          // rays from pixels / world points -> camera frame, once per upload, in place
    BuildArgs ba{};
    ba.meta = reinterpret_cast<ObjMeta*>(db + o_meta); ba.T_init = reinterpret_cast<float*>(db + o_T);
    ba.pts = reinterpret_cast<float*>(db + o_pts); ba.rays = reinterpret_cast<float*>(db + o_rays);
    ba.aux = reinterpret_cast<const float*>(db + o_aux); ba.n_obj = n_obj;
    k_build_inputs<<<n_obj, 256, 0, s->stream>>>(ba);
    CU(cudaGetLastError());
  }
  if (grid_dim) {
    if (s->d_grid_pts.cap < 12 * (size_t)tp) CU(settle_stream(s));
    if (s->d_grid_pts.reserve(12 * (size_t)tp)) return fail(DSPGN_E_ALLOC, "grid allocation failed");
    const long long R = (long long)grid_dim * grid_dim * grid_dim;
    k_mesh_grid_points<<<dim3((unsigned)((R + 255) / 256), (unsigned)std::min(n_obj, 65535)), 256, 0, s->stream>>>(
        s->d_grid_pts.as<float>(), n_obj, grid_dim);
    s->ctr.kernel_launches++;
    CU(cudaGetLastError());
  }
  s->d_meta = reinterpret_cast<ObjMeta*>(db + o_meta);
  s->d_Tinit = reinterpret_cast<float*>(db + o_T);
  s->d_code = reinterpret_cast<float*>(db + o_code);
  s->d_pts = grid_dim ? s->d_grid_pts.as<float>() : reinterpret_cast<float*>(db + o_pts);
  s->d_rays = reinterpret_cast<float*>(db + o_rays);
  s->d_depth = reinterpret_cast<float*>(db + o_depth);
  s->d_tbase_static = reinterpret_cast<int*>(db + o_tb);
  s->d_tbase_r_static = s->d_tbase_static + n_obj;
  s->run_table_valid = false;
  s->n_obj = n_obj; s->tot_pts = (int)tp; s->tot_rays = (int)tr; s->tot_fg = (int)tf; s->tot_smp = ts; s->max_rays = max_rays;
  s->gather.bound_n = -1;
  int bad = 0;
  bad |= s->d_state.reserve(sizeof(ObjState) * n_obj);
  const bool render = !decode_only && !s->cfg.sdf_only;
  if (!decode_only) {
    // per-tile partial sums: one slot per possible tile of each term at the engine's tile height
    const size_t rows_per_tile = tile_rows(s);
    const size_t tiles_s = (size_t)tp / rows_per_tile + n_obj + 1, tiles_r = (size_t)ts / rows_per_tile + 2 * (size_t)n_obj + 1;
    bad |= s->d_part_s.reserve(4 * (size_t)kAccStride * tiles_s);
    if (render) bad |= s->d_part_r.reserve(4 * (size_t)kAccStride * tiles_r);
    bad |= s->d_active.reserve((size_t)tp + 1);
  }
  bad |= s->d_tbase.reserve(4 * 2 * (size_t)n_obj);
  bad |= s->d_V.reserve(4 * (size_t)n_obj);
  bad |= s->d_m.reserve(4 * (size_t)n_obj);
  bad |= s->d_results.reserve(4 * DSPGN_RESULT_FLOATS * (size_t)n_obj);
  bad |= s->h_results.reserve(4 * DSPGN_RESULT_FLOATS * (size_t)n_obj + 512);
  const size_t smp = (size_t)(ts > 0 ? ts : 1);
  if (render) {
    bad |= s->d_sdf.reserve(4 * smp);
    bad |= s->d_bx.reserve(12 * smp);
    bad |= s->d_bs.reserve(4 * smp);
    bad |= s->d_br.reserve(4 * smp);
  }
  bad |= s->d_dbg.reserve(4 * ((size_t)kPMax * kPMax + 2 * kPMax + 8));
  if (bad) return fail(DSPGN_E_ALLOC, "workspace allocation failed");
  return 0;
}

}  // namespace

int dspgn_upload_batch(DspgnSolver* s, int n_obj, const DspgnObjectIn* in) {
  BUSY(s);
  return upload_batch_impl(s, n_obj, in, false);
}

namespace {

cudaEvent_t next_event(DspgnSolver* s) {
  if (s->ev_used == s->ev.size()) { cudaEvent_t e; cudaEventCreate(&e); s->ev.push_back(e); }
  return s->ev[s->ev_used++];
}

int launch_term(DspgnSolver* s, const BatchDev& b, const TermArgs& a, long long rows_upper, cudaStream_t stream = nullptr,
                bool use_given = false) {
  cudaStream_t st = use_given ? stream : s->stream;
  const bool timed = s->timing && !use_given;
  if (timed) cudaEventRecord(next_event(s), st);
  const long long rows = tile_rows(s);
  long long tiles = (rows_upper + rows - 1) / rows + s->n_obj;
  if (s->engine == DSPGN_ENGINE_TC) {
    if (int rc = tc_launch_term(b, a, grid_sms(s), tiles, st, g_err)) return rc;
  } else if (s->engine == DSPGN_ENGINE_TC_WIDE) {
    tcw_launch_term(b, a, s->d_tcw.as<TcwDecDev>(), s->d_masks.as<uint4>(), grid_sms(s), tiles, st);
  } else {
    int grid = (int)std::min<long long>(tiles, grid_sms(s));
    if (grid < 1) grid = 1;
    if (s->simt_hid == kHid) k_decoder_simt<kHid><<<grid, kThreads, sizeof(SimtSmem<kHid>), st>>>(b, a);
    else k_decoder_simt<kHidWide><<<grid, kThreads, sizeof(SimtSmem<kHidWide>), st>>>(b, a);
  }
  if (timed) cudaEventRecord(next_event(s), st);
  s->ctr.kernel_launches++;
  CU(cudaGetLastError());
  return 0;
}

TermArgs base_term(DspgnSolver* s, int mode) {
  TermArgs a{};
  a.mode = mode;
  a.pt_active = nullptr; a.cut_iter = -1; a.iter = 0;
  a.part = (mode == MODE_BAND) ? s->d_part_r.as<float>() : (mode == MODE_SDF ? s->d_part_s.as<float>() : nullptr);
  a.tile_base = (mode == MODE_BAND) ? s->d_tbase.as<int>() + s->n_obj : (mode == MODE_SDF ? s->d_tbase.as<int>() : nullptr);
  a.ln_scratch = s->d_ln.p ? s->d_ln.as<float>() + (mode == MODE_RAYFWD ? ln_half_floats(s) : 0) : nullptr;
  a.dbg_J = nullptr; a.dbg_res = nullptr; a.dbg_obj = -1; a.dbg_P = 0;
  return a;
}

// The per-run object table, staged in h_run and copied to d_run: modes [n] | first iteration-0 queue slot of the
// persistent kernel [n] | link [n] | t_map [n][16] (the last two in a gated run only).
struct RunTable { int* modes; int* q0_off; int* link; float* t_map; };
size_t run_table_bytes(int n, bool gated) { return (gated ? 12 + 64 : 8) * (size_t)n; }
RunTable run_table(void* base, int n, bool gated) {
  int* p = static_cast<int*>(base);
  return RunTable{p, p + n, gated ? p + 2 * n : nullptr, gated ? reinterpret_cast<float*>(p + 3 * n) : nullptr};
}

// What the caller of a run passes its kernels besides the resident batch: the multi-GPU exchange slots
// (dspgn_run_batch_gather) and, for a chunk of a stoppable call, the chunk's slot of the call's stop hook and the pair
// partners of its slots on the device (meshed calls with pairs).
struct RunArgs {
  GatherDev gather{};                // slots == nullptr: no exchange
  int stop_slot = -1;                // resident slot of call_stop_obj (-1: not in this chunk)
  const int* pair = nullptr;
};

// The resident batch and its run table as the kernels see them.  Call after plan_run (it may move d_run) and after
// every buffer reservation of the run.
BatchDev batch_dev(DspgnSolver* s, const RunArgs& r) {
  BatchDev b{};
  b.meta = s->d_meta; b.state = s->d_state.as<ObjState>(); b.decs = s->d_decs.as<DecoderDev>();
  b.n_obj = s->n_obj; b.n_classes = (int)s->classes.size(); b.D = s->cfg.num_depth_samples;
  b.pts = s->d_pts; b.rays = s->d_rays; b.depth_fg = s->d_depth; b.T_init = s->d_Tinit; b.code_init = s->d_code;
  b.sdf = s->d_sdf.as<float>(); b.band_x = s->d_bx.as<float>(); b.band_s = s->d_bs.as<float>(); b.band_r = s->d_br.as<float>();
  b.band_m = s->d_m.as<int>(); b.V_count = s->d_V.as<int>();
  b.results = s->d_results.as<float>();
  b.gather = r.gather;
  const RunTable t = run_table(s->d_run.p, s->n_obj, s->run_table_gated);
  b.modes = t.modes; b.q0_off = t.q0_off; b.link = t.link; b.t_map = t.t_map;
  // only the runs of a stoppable call can stop, and never those of the multi-GPU exchange
  const bool stoppable = s->stop_live.load(std::memory_order_relaxed) != 0 && r.gather.slots == nullptr;
  b.stop = stoppable ? StopDev{s->d_stop, s->stop_gen, r.stop_slot, s->call_stop_iter, r.pair}
                     : StopDev{nullptr, 0u, -1, -1, nullptr};
  b.lin = s->lin_base >= 0 ? s->d_lin.as<float>() + (size_t)s->lin_base * lin_floats(s->cfg.code_len) : nullptr;
  return b;
}

// ---- pose information (dspgn_pose_information) ----------------------------------------------------------------------
// A call that returns records keeps the last linearisation of each of its `slots` slots (all chunks) in d_lin, the chunk
// at lin_base; the scope ends it.  d_lin grows like the batch's other buffers (d_results: no settle, cudaFree waits).
struct LinScope {
  DspgnSolver* s;
  explicit LinScope(DspgnSolver* s_) : s(s_) {}
  ~LinScope() { s->lin_base = -1; }
  int begin(size_t slots, size_t n_obj) {
    s->info_valid = false;
    s->info_items.assign(n_obj, InfoItem{-1, 0, 0.0});
    if (s->d_lin.reserve(4 * (size_t)lin_floats(s->cfg.code_len) * slots)) return fail(DSPGN_E_ALLOC, "linearisation buffer allocation failed");
    s->lin_base = 0;
    return 0;
  }
};

// The item of a record from call slot `slot`; pose_scale > 0: a pose-only record whose solver pose carried that scale
// (estimate_pose_cam_obj's argument), else a joint record, whose scale is cbrt(det R) of its pose as
// SetPoseMeasurementSim3 takes it.  Only a record whose final update came from a completed solve has a linearisation.
InfoItem info_item(const DspgnSolver* s, const DspgnObjectOut& r, int slot, float pose_scale) {
  InfoItem it{-1, 0, 0.0};
  if ((r.status != DSPGN_ST_OK && r.status != DSPGN_ST_STOPPED) || r.iters_done < 1) return it;
  const float* T = r.t_cam_obj;
  const double det = (double)T[0] * ((double)T[5] * T[10] - (double)T[6] * T[9]) -
                     (double)T[1] * ((double)T[4] * T[10] - (double)T[6] * T[8]) +
                     (double)T[2] * ((double)T[4] * T[9] - (double)T[5] * T[8]);
  it.slot = slot;
  it.P = pose_scale > 0.f ? 6 : 7 + s->cfg.code_len;
  it.s = pose_scale > 0.f ? (double)pose_scale : std::cbrt(det);
  return it;
}

// What a run does with the resident batch, given one mode per object: iteration counts and row counters per mode, and
// the work queue of the persistent kernel (capacity, iteration-0 slots).  A uniform mode array is dspgn_run_batch(s, m).
struct RunPlan {
  int iters[2];            // GN iterations of a joint / pose-only object
  bool any[2];             // the run has objects of this mode
  bool render;             // the joint objects run the render term
  long long pts[2];        // surface points of the objects of each mode
  long long smp_joint;     // ray samples (n_rays x D) of the joint objects
  long long q_cap;         // persistent kernel: work items that can ever be pushed
  int total0;              // persistent kernel: iteration-0 queue slots (k_init seeds them)
  bool gated;              // the run table carries link | t_map (a gated keyframe run)
  bool any_dormant;        // ... and has joint slots that only run when their pose-only object is rejected
};

// Checks the modes, fills the plan and stages the per-run object table (run_table) into d_run, async on the stream;
// `unlimited`: objects never finish (the debug
// hooks advance the batch freely).  link[o] >= 0 on a joint object marks the dormant joint slot of pose-only object
// link[o]: it counts towards the queue capacity and the render term but reserves no iteration-0 slot and no row counter.
int plan_run(DspgnSolver* s, const int32_t* modes, RunPlan& p, bool unlimited = false, const int32_t* link = nullptr,
             const float* t_map = nullptr) {
  const DspgnConfig& c = s->cfg;
  const int n = s->n_obj, D = c.num_depth_samples, rows = tile_rows(s);
  p = RunPlan{};
  p.gated = link != nullptr;
  for (int o = 0; o < n; ++o) {
    if (modes[o] != DSPGN_MODE_JOINT && modes[o] != DSPGN_MODE_POSE) return fail(DSPGN_E_ARG, "mode must be 0 or 1");
    if (link && link[o] >= 0 && modes[o] == DSPGN_MODE_JOINT) p.any_dormant = true;
    else p.any[modes[o]] = true;
  }
  if (p.any[DSPGN_MODE_POSE] && c.pose_only_iterations < 1) return fail(DSPGN_E_ARG, "pose_only_iterations must be >= 1");
  p.iters[DSPGN_MODE_JOINT] = unlimited ? (1 << 30) : c.num_iterations;
  p.iters[DSPGN_MODE_POSE] = unlimited ? (1 << 30) : c.pose_only_iterations;
  p.render = (p.any[DSPGN_MODE_JOINT] || p.any_dormant) && !c.sdf_only;
  if (s->run_upload_pending) { CU(settle_event(s, s->ev_run_upload)); s->run_upload_pending = false; }
  const size_t bytes = run_table_bytes(n, p.gated);
  const bool same = s->run_table_valid && !p.gated && !s->run_table_gated &&
                    memcmp(run_table(s->h_run.p, n, false).modes, modes, 4 * (size_t)n) == 0;
  if (!same) {
    if (s->d_run.cap < bytes) CU(settle_stream(s));      // kernels of an earlier run may still read it
    if (s->h_run.reserve(bytes) || s->d_run.reserve(bytes)) return fail(DSPGN_E_ALLOC, "run table allocation failed");
  }
  const RunTable h = run_table(s->h_run.p, n, p.gated);
  for (int o = 0; o < n; ++o) {
    const ObjMeta& M = s->h_meta[o];
    const int m = modes[o];
    const bool dormant = link && link[o] >= 0 && m == DSPGN_MODE_JOINT;
    const bool r = p.render && m == DSPGN_MODE_JOINT;
    const auto [ntS, ntF] = obj_tiles(M, D, rows);
    if (!dormant) {
      p.pts[m] += M.n_pts;
      if (m == DSPGN_MODE_JOINT) p.smp_joint += (long long)M.n_rays * D;
    }
    // per iteration: every SDF tile, every ray-sample tile, one scan item per 64 rays and at most as many band tiles
    // as ray-sample tiles (iteration 0 reserves every ray-sample tile of the object)
    p.q_cap += (long long)p.iters[m] * (ntS + (r ? 2 * ntF + (M.n_rays + kScanChunkRays - 1) / kScanChunkRays : 0));
    if (!same) { h.modes[o] = m; h.q0_off[o] = p.total0; }
    if (!dormant) p.total0 += (int)(ntS + (r ? ntF : 0));
  }
  if (p.gated) {
    memcpy(h.link, link, 4 * (size_t)n);
    memcpy(h.t_map, t_map, 64 * (size_t)n);
  }
  s->run_table_gated = p.gated;
  if (!same) {
    CU(cudaMemcpyAsync(s->d_run.p, s->h_run.p, bytes, cudaMemcpyHostToDevice, s->stream));
    CU(cudaEventRecord(s->ev_run_upload, s->stream));
    s->run_upload_pending = true;
    s->run_table_valid = true;
  }
  return 0;
}

// q: the persistent kernel's queue (mega_args) when it runs next, else empty
int launch_init(DspgnSolver* s, const BatchDev& b, const RunPlan& p, const MegaArgs& q = MegaArgs{}) {
  InitArgs ia{};
  ia.code_len = s->cfg.code_len;
  ia.n_iter_joint = p.iters[DSPGN_MODE_JOINT]; ia.n_iter_pose = p.iters[DSPGN_MODE_POSE];
  ia.n_bad = s->n_bad;
  ia.tile_rows = tile_rows(s);
  k_init<<<s->n_obj, 128, 0, s->stream>>>(b, ia, q);
  s->ctr.kernel_launches++;
  CU(cudaGetLastError());
  return 0;
}

// one GN iteration's residual-term kernels (everything before the solve); objects past their own last iteration
// contribute no rows
int launch_terms(DspgnSolver* s, const BatchDev& b, const RunPlan& p, int iter, float* dbg_J = nullptr, float* dbg_res = nullptr,
                 int dbg_obj = -1, int dbg_P = 0) {
  const DspgnConfig& c = s->cfg;
  const bool render = p.render && p.any[DSPGN_MODE_JOINT] && iter < p.iters[DSPGN_MODE_JOINT];
  // The SDF-row pass and the forward-only pass over the ray samples are independent: fork the latter onto a
  // second stream (matters for small batches, where each pass is a single wave of tiles) unless per-launch
  // timing is on.
  const bool fork = render && !s->timing;
  if (render) {
    TermArgs f = base_term(s, MODE_RAYFWD);
    f.iter = iter;
    if (fork) {
      CU(cudaEventRecord(s->ev_fork, s->stream));
      CU(cudaStreamWaitEvent(s->stream2, s->ev_fork, 0));
      if (int rc = launch_term(s, b, f, s->tot_smp, s->stream2, true)) return rc;
      CU(cudaEventRecord(s->ev_join, s->stream2));
    } else {
      if (int rc = launch_term(s, b, f, s->tot_smp)) return rc;
    }
    s->ctr.rows_fwd_only += p.smp_joint;
  }
  {
    TermArgs a = base_term(s, MODE_SDF);
    a.huber_b = c.b2;                                  // pose-only objects: raw residuals (optimizer.py:71, term_huber)
    a.iter = iter;
    a.pt_active = s->d_active.as<uint8_t>(); a.cut_iter = 4;   // optimizer.py:76-78: inlier cut taken after iteration index 4
    a.dbg_J = dbg_J; a.dbg_res = dbg_res; a.dbg_obj = dbg_obj; a.dbg_P = dbg_P;
    if (int rc = launch_term(s, b, a, s->tot_pts)) return rc;
    for (int m = 0; m < 2; ++m)
      if (iter < p.iters[m]) s->ctr.rows_fwd_bwd += p.pts[m];
  }
  if (render) {
    if (fork) CU(cudaStreamWaitEvent(s->stream, s->ev_join, 0));
    k_ray_scan<<<s->n_obj, kScanThreads, 0, s->stream>>>(b, c.cut_off);
    s->ctr.kernel_launches++;
    CU(cudaGetLastError());
    TermArgs band = base_term(s, MODE_BAND);
    band.huber_b = c.b1;
    band.iter = iter;
    if (int rc = launch_term(s, b, band, s->tot_smp)) return rc;
  }
  return 0;
}

SolveArgs base_solve(DspgnSolver* s) {
  const DspgnConfig& c = s->cfg;
  SolveArgs v{};
  v.part_s = s->d_part_s.as<float>(); v.part_r = s->d_part_r.as<float>();
  v.base_s = s->d_tbase.as<int>(); v.base_r = s->d_tbase.as<int>() + s->n_obj;
  v.tile_rows = tile_rows(s);
  v.prm = SolverParams{c.k1, c.k2, c.k3, c.k4, c.b1, c.b2, c.lr, c.s_damp, c.code_len, c.num_depth_samples, c.cut_off, c.sdf_only};
  v.dbg_obj = -1; v.dbg_H = nullptr; v.dbg_b = nullptr; v.dbg_dx = nullptr; v.dbg_loss = nullptr;
  return v;
}

// The solve of GN iteration v.iter_index (per-iteration schedule), timed in ev_solve when timing is on
int launch_solve(DspgnSolver* s, const BatchDev& b, const SolveArgs& v) {
  if (s->timing) {
    if (s->evs_used + 2 > s->ev_solve.size()) { cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1); s->ev_solve.push_back(e0); s->ev_solve.push_back(e1); }
    cudaEventRecord(s->ev_solve[s->evs_used], s->stream);
  }
  k_solve<<<s->n_obj, kSolveThreads, 0, s->stream>>>(b, v);
  if (s->timing) { cudaEventRecord(s->ev_solve[s->evs_used + 1], s->stream); s->evs_used += 2; }
  s->ctr.kernel_launches++;
  CU(cudaGetLastError());
  return 0;
}

// GN iterations 0 .. n_iters - 1 of plan p on the per-iteration schedule: each one's terms, then its solve
int gn_iterations(DspgnSolver* s, const BatchDev& b, const RunPlan& p, int n_iters) {
  for (int e = 0; e < n_iters; ++e) {
    if (int rc = launch_terms(s, b, p, e)) return rc;
    SolveArgs v = base_solve(s);
    v.iter_index = e;
    if (int rc = launch_solve(s, b, v)) return rc;
  }
  return 0;
}

// The persistent kernel's work queue for the run: reserves its buffers and builds its MegaArgs (k_init seeds it, the
// kernel runs on it).
int mega_args(DspgnSolver* s, const RunPlan& p, MegaArgs& q) {
  const bool render = p.render;
  const int cap = (int)p.q_cap;
  const int n = s->n_obj;
  const size_t nseg_cap = (size_t)s->tot_rays / kSegRays + 2 * (size_t)n + 4;
  int bad = 0;
  bad |= s->d_q_flag.reserve(4 * (size_t)cap);
  bad |= s->d_q_ctr.reserve(sizeof(QueueCounters));
  bad |= s->d_tiles_left.reserve(4 * 3 * (size_t)n);
  if (render) bad |= s->d_seg.reserve(4 * 2 * nseg_cap);
  if (render && s->compact_rays) bad |= s->d_vpre.reserve(4 * ((size_t)s->tot_rays + (size_t)n + 4));
  bad |= s->d_obj_iter.reserve(4 * (size_t)n);
  if (s->events_on) bad |= s->d_ev.reserve(8 * (1 + 2 * (size_t)kEvCap));
  if (bad) return fail(DSPGN_E_ALLOC, "queue allocation failed");
  q = MegaArgs{};
  q.q_cap = cap; q.render = render ? 1 : 0; q.total0 = p.total0;
  q.q_flag = s->d_q_flag.as<int>();
  q.ctr = s->d_q_ctr.as<QueueCounters>();
  q.pending = s->d_tiles_left.as<int>(); q.ray_left = s->d_tiles_left.as<int>() + n; q.scan_left = s->d_tiles_left.as<int>() + 2 * n;
  q.seg_cnt = s->d_seg.as<int>(); q.seg_prefix = s->d_seg.as<int>() + nseg_cap;
  q.obj_iter = s->d_obj_iter.as<int>();
  q.vpre = (render && s->compact_rays) ? s->d_vpre.as<int>() : nullptr;
  if (s->events_on) q.log = EventLog{s->d_ev.as<long long>(), kEvCap};
  return 0;
}

}  // namespace

namespace {
// One run of the resident batch, modes[o] = DSPGN_MODE_* of object o.  Every object runs its own mode's iterations,
// terms and update and finishes after its own last iteration; dspgn_run_batch(s, m) is the uniform case.
// A gated run (link != nullptr, see plan_run) also checks every gated pose-only object at its last solve and runs the joint
// slots of the rejected ones: woken on the device by the persistent kernel; in the per-iteration schedule as a second
// phase after a readback of the verdicts, or (device_wake, a submitted call) as a second phase enqueued for every gated
// slot: k_gate_wake reads the verdicts itself and the slots it does not wake have n_iter 0, so they contribute no rows
// (term_rows) and k_solve skips them -- the same records.  Their rows are counted when the records come back.
int run_batch_impl(DspgnSolver* s, const int32_t* modes, const RunArgs& ra, const int32_t* link = nullptr,
                   const float* t_map = nullptr, bool device_wake = false) {
  CU(cudaSetDevice(s->device));
  RunPlan p;
  if (int rc = plan_run(s, modes, p, false, link, t_map)) return rc;
  const BatchDev b = batch_dev(s, ra);
  const int max_iters = std::max(p.any[DSPGN_MODE_JOINT] ? p.iters[DSPGN_MODE_JOINT] : 0,
                                 p.any[DSPGN_MODE_POSE] ? p.iters[DSPGN_MODE_POSE] : 0);
  if (int rc = run_begin(s)) return rc;
  const bool render = p.render;
  const bool wide = s->engine == DSPGN_ENGINE_TC_WIDE, simt = s->engine == DSPGN_ENGINE_SIMT;
  const bool mega = s->mega_enabled && s->total_tiles > 0 &&
                    s->max_tiles <= kItemTileMask && s->n_obj <= kItemObjMask + 1 && p.q_cap < (1LL << 27);
  if (mega) {
    // ---- persistent object-pipelined kernel: every GN iteration of every object in ONE launch --------------
    MegaArgs q;
    if (int rc = mega_args(s, p, q)) return rc;
    CU(cudaMemsetAsync(q.q_flag, 0, 4 * (size_t)q.q_cap, s->stream));
    if (int rc = launch_init(s, b, p, q)) return rc;
    TermArgs a = base_term(s, MODE_SDF);
    a.huber_b = s->cfg.b2;                   // pose-only objects: raw residuals (term_huber)
    a.huber_b1 = s->cfg.b1;
    a.tile_base = s->d_tbase_static;
    a.part_r = s->d_part_r.as<float>(); a.tile_base_r = s->d_tbase_r_static;
    if (p.any[DSPGN_MODE_POSE] && p.iters[DSPGN_MODE_POSE] > 5) { a.pt_active = s->d_active.as<uint8_t>(); a.cut_iter = 4; }
    if (q.log.ev) CU(cudaMemsetAsync(q.log.ev, 0, 8, s->stream));
    SolveArgs v = base_solve(s);
    v.base_s = s->d_tbase_static; v.base_r = s->d_tbase_r_static; v.iter_index = 0;
    const int grid = grid_sms(s);
    if (s->timing) cudaEventRecord(next_event(s), s->stream);
    if (simt && s->simt_hid == kHid) k_simt_persistent<kHid><<<grid, kThreads, sizeof(SimtMegaSmem<kHid>), s->stream>>>(b, a, q, v);
    else if (simt) k_simt_persistent<kHidWide><<<grid, kThreads, sizeof(SimtMegaSmem<kHidWide>), s->stream>>>(b, a, q, v);
    else if (wide) k_wide_persistent<<<grid, kTcThreads, kTcwMegaSmemBytes, s->stream>>>(b, a, q, v, s->d_tcw.as<TcwDecDev>(), s->d_masks.as<uint4>());
    else if (render) k_gn_persistent_render<<<grid, kTcThreads, kTcSmemBytes<2>, s->stream>>>(b, a, q, v);
    else k_gn_persistent<<<grid, kTcThreads, kTcSmemBytes<1>, s->stream>>>(b, a, q, v, s->d_masks.as<uint4>());
    if (s->timing) cudaEventRecord(next_event(s), s->stream);
    s->ctr.kernel_launches += 1;
    for (int m = 0; m < 2; ++m) s->ctr.rows_fwd_bwd += p.pts[m] * p.iters[m];
    s->band_rows_pending = render;           // band rows and valid ray samples are counted by the kernel (dspgn_results)
    s->mega_ran = true;
    CU(cudaGetLastError());
    return run_end(s);
  }
  if (int rc = launch_init(s, b, p)) return rc;
  if (int rc = gn_iterations(s, b, p, max_iters)) return rc;
  if (p.any_dormant && device_wake) {
    RunPlan pb = p;
    pb.any[DSPGN_MODE_POSE] = false; pb.any[DSPGN_MODE_JOINT] = true;
    pb.pts[DSPGN_MODE_POSE] = 0; pb.pts[DSPGN_MODE_JOINT] = 0; pb.smp_joint = 0;
    k_gate_wake<<<(s->n_obj + 127) / 128, 128, 0, s->stream>>>(b, p.iters[DSPGN_MODE_JOINT]);
    s->ctr.kernel_launches++;
    CU(cudaGetLastError());
    if (int rc = gn_iterations(s, b, pb, pb.iters[DSPGN_MODE_JOINT])) return rc;
  } else if (p.any_dormant) {
    // second phase: the verdicts of the first (record gate words) decide which joint slots run
    const int n = s->n_obj;
    if (s->h_results.reserve(4 * DSPGN_RESULT_FLOATS * (size_t)n + 512)) return fail(DSPGN_E_ALLOC, "cudaMallocHost");
    CU(cudaMemcpyAsync(s->h_results.p, s->d_results.p, 4 * DSPGN_RESULT_FLOATS * (size_t)n, cudaMemcpyDeviceToHost, s->stream));
    CU(sync_stream(s));
    const int* rec = s->h_results.as<int>();
    RunPlan pb = p;
    pb.any[DSPGN_MODE_POSE] = false; pb.any[DSPGN_MODE_JOINT] = false;
    pb.pts[DSPGN_MODE_POSE] = 0; pb.pts[DSPGN_MODE_JOINT] = 0; pb.smp_joint = 0;
    for (int o = 0; o < n; ++o)
      if (link[o] >= 0 && modes[o] == DSPGN_MODE_JOINT && rec[(size_t)link[o] * DSPGN_RESULT_FLOATS + 85] == DSPGN_GATE_REJECTED) {
        pb.any[DSPGN_MODE_JOINT] = true;
        pb.pts[DSPGN_MODE_JOINT] += s->h_meta[o].n_pts;
        pb.smp_joint += (long long)s->h_meta[o].n_rays * s->cfg.num_depth_samples;
      }
    if (pb.any[DSPGN_MODE_JOINT]) {
      k_gate_wake<<<(n + 127) / 128, 128, 0, s->stream>>>(b, p.iters[DSPGN_MODE_JOINT]);
      s->ctr.kernel_launches++;
      CU(cudaGetLastError());
      if (int rc = gn_iterations(s, b, pb, pb.iters[DSPGN_MODE_JOINT])) return rc;
    }
  }
  return run_end(s);
}

// dspgn_run_batch / dspgn_run_batch_gather / the whole-batch calls: every object in `mode`
int run_uniform(DspgnSolver* s, int mode, const RunArgs& ra) {
  if (!s) return fail(DSPGN_E_ARG, "null solver");
  if (s->n_obj < 1) return fail(DSPGN_E_ARG, "no batch uploaded");
  if (mode != DSPGN_MODE_JOINT && mode != DSPGN_MODE_POSE) return fail(DSPGN_E_ARG, "mode must be 0 or 1");
  const std::vector<int32_t> modes(s->n_obj, mode);
  return run_batch_impl(s, modes.data(), ra);
}

// call-level misuse of the per-object entry points: modes outside {0, 1}; a pose-only object without a code or with
// scale <= 0 (estimate_pose_cam_obj's arguments, checked like dspgn_estimate_pose_batch does).  The objects are the
// caller's `in` or, when it is null, the resident batch.
int check_modes(const DspgnSolver* s, const int32_t* modes, int n, const DspgnObjectIn* in) {
  for (int o = 0; o < n; ++o) {
    if (modes[o] != DSPGN_MODE_JOINT && modes[o] != DSPGN_MODE_POSE) return fail(DSPGN_E_ARG, "mode must be 0 or 1");
    const bool code = in ? in[o].code != nullptr : s->h_meta[o].has_code != 0;
    const float scale = in ? in[o].scale : s->h_meta[o].scale;
    if (modes[o] == DSPGN_MODE_POSE && (!code || !(scale > 0.f)))
      return fail(DSPGN_E_ARG, "a pose-only object needs a code and a positive scale");
  }
  return 0;
}

GatherDev gather_dev(DspgnSolver* s, int seq) {
  DspgnSolver::Gather& G = s->gather;
  GatherDev g{};
  g.slots = reinterpret_cast<float*>(G.base) + (size_t)(seq & 1) * G.n_slots * DSPGN_RESULT_FLOATS;
  g.slot_of = G.d_slot_of.as<int>();
  g.flags = reinterpret_cast<int*>(G.base + G.off_flags);
  g.ack = reinterpret_cast<int*>(G.base + G.off_ack);
  g.err = G.d_local.as<int>();
  g.wait_ns = reinterpret_cast<long long*>(G.d_local.as<unsigned char>() + 8);
  g.rank = G.rank; g.world = G.world; g.seq = seq;
  return g;
}

int gather_layout(DspgnSolver* s, int n_slots, int world, int rank) {
  DspgnSolver::Gather& G = s->gather;
  G.n_slots = n_slots; G.world = world; G.rank = rank;
  const size_t slot_bytes = 2 * (size_t)n_slots * DSPGN_RESULT_FLOATS * 4;
  G.off_flags = (slot_bytes + 255) / 256 * 256;
  G.off_ack = G.off_flags + 4 * (size_t)((world + 63) / 64 * 64);
  if (G.d_local.reserve(64)) return fail(DSPGN_E_ALLOC, "cudaMalloc");
  CU(cudaMemset(G.d_local.p, 0, 64));
  return 0;
}
}  // namespace

int dspgn_run_batch(DspgnSolver* s, int mode) {
  BUSY(s);
  return run_uniform(s, mode, RunArgs{});
}

int dspgn_run_batch_modes(DspgnSolver* s, const int32_t* modes) {
  if (!s || !modes) return fail(DSPGN_E_ARG, "null argument");
  BUSY(s);
  if (s->n_obj < 1) return fail(DSPGN_E_ARG, "no batch uploaded");
  if (int rc = check_modes(s, modes, s->n_obj, nullptr)) return rc;
  return run_batch_impl(s, modes, RunArgs{});
}

// ---- multi-GPU result exchange ----------------------------------------------------------------------------------
int dspgn_gather_create(DspgnSolver* s, int n_slots, int world, DspgnIpcHandle* handle_out) {
  if (!s || !handle_out || n_slots < 1 || world < 1 || world > 1024) return fail(DSPGN_E_ARG, "bad gather arguments");
  BUSY(s);
  static_assert(sizeof(cudaIpcMemHandle_t) <= DSPGN_IPC_HANDLE_BYTES, "IPC handle size");
  CU(cudaSetDevice(s->device));
  dspgn_gather_close(s);
  if (int rc = gather_layout(s, n_slots, world, 0)) return rc;
  DspgnSolver::Gather& G = s->gather;
  const size_t bytes = G.off_ack + 256;
  void* p = nullptr;
  CU(cudaMalloc(&p, bytes));           // plain cudaMalloc: exportable through cudaIpcGetMemHandle
  G.base = reinterpret_cast<unsigned char*>(p); G.owner = true;
  CU(cudaMemset(p, 0, bytes));
  cudaIpcMemHandle_t h;
  memset(handle_out, 0, sizeof(*handle_out));
  if (world > 1) {
    CU(cudaIpcGetMemHandle(&h, p));
    memcpy(handle_out->bytes, &h, sizeof(h));
  }
  G.active = true;
  return 0;
}

int dspgn_gather_open(DspgnSolver* s, const DspgnIpcHandle* handle, int n_slots, int world, int rank) {
  if (!s || !handle || n_slots < 1 || world < 2 || rank < 1 || rank >= world) return fail(DSPGN_E_ARG, "bad gather arguments");
  BUSY(s);
  CU(cudaSetDevice(s->device));
  dspgn_gather_close(s);
  if (int rc = gather_layout(s, n_slots, world, rank)) return rc;
  DspgnSolver::Gather& G = s->gather;
  cudaIpcMemHandle_t h;
  memcpy(&h, handle->bytes, sizeof(h));
  void* p = nullptr;
  CU(cudaIpcOpenMemHandle(&p, h, cudaIpcMemLazyEnablePeerAccess));   // rank 0's HBM, reachable over NVLink
  G.base = reinterpret_cast<unsigned char*>(p); G.owner = false;
  G.active = true;
  return 0;
}

void dspgn_gather_close(DspgnSolver* s) {
  if (!s) return;
  if (s->flight.active) { fail(DSPGN_E_BUSY, "a submitted keyframe call is in flight"); return; }
  DspgnSolver::Gather& G = s->gather;
  if (G.base) {
    cudaSetDevice(s->device);
    sync_stream(s);
    if (G.owner) cudaFree(G.base); else cudaIpcCloseMemHandle(G.base);
    cudaGetLastError();
  }
  G.base = nullptr; G.active = false; G.owner = false; G.bound_n = -1;
  G.d_slot_of.release(); G.d_local.release(); G.h_out.release();
}

int dspgn_gather_bind(DspgnSolver* s, const int32_t* slots, int n) {
  if (!s || n < 0 || (n > 0 && !slots)) return fail(DSPGN_E_ARG, "bad argument");
  BUSY(s);
  DspgnSolver::Gather& G = s->gather;
  if (!G.active) return fail(DSPGN_E_ARG, "no gather buffer (dspgn_gather_create / dspgn_gather_open first)");
  if (n > 0 && n != s->n_obj) return fail(DSPGN_E_ARG, "gather_bind: n must equal the resident batch size");
  for (int i = 0; i < n; ++i)
    if (slots[i] < 0 || slots[i] >= G.n_slots) return fail(DSPGN_E_ARG, "gather_bind: slot out of range");
  CU(cudaSetDevice(s->device));
  if (n > 0) {
    if (G.d_slot_of.cap < 4 * (size_t)n) CU(settle_stream(s));
    if (G.d_slot_of.reserve(4 * (size_t)n)) return fail(DSPGN_E_ALLOC, "cudaMalloc");
    CU(cudaMemcpyAsync(G.d_slot_of.p, slots, 4 * (size_t)n, cudaMemcpyHostToDevice, s->stream));   // pageable source: returns after staging
  }
  G.bound_n = n;
  return 0;
}

int dspgn_run_batch_gather(DspgnSolver* s, int mode, int seq) {
  if (!s || seq < 1) return fail(DSPGN_E_ARG, "bad argument");
  BUSY(s);
  DspgnSolver::Gather& G = s->gather;
  if (!G.active || G.bound_n < 0) return fail(DSPGN_E_ARG, "gather not bound for the resident batch");
  CU(cudaSetDevice(s->device));
  const GatherDev g = gather_dev(s, seq);
  if (G.bound_n > 0)
    if (int rc = run_uniform(s, mode, RunArgs{g})) return rc;
  k_gather_publish<<<1, 32, 0, s->stream>>>(g, G.bound_n == 0 ? 1 : 0);
  if (G.rank == 0) k_gather_wait<<<1, 32 * ((G.world + 31) / 32), 0, s->stream>>>(g);
  s->ctr.kernel_launches += (G.rank == 0) ? 2 : 1;
  CU(cudaGetLastError());
  return 0;
}

const float* dspgn_gather_device(DspgnSolver* s, int seq) {
  if (!s || !s->gather.active) return nullptr;
  if (s->flight.active) { fail(DSPGN_E_BUSY, "a submitted keyframe call is in flight"); return nullptr; }
  return reinterpret_cast<const float*>(s->gather.base) + (size_t)(seq & 1) * s->gather.n_slots * DSPGN_RESULT_FLOATS;
}

int dspgn_gather_results(DspgnSolver* s, int seq, int n, DspgnObjectOut* out) {
  if (!s || !out || n < 1) return fail(DSPGN_E_ARG, "bad argument");
  BUSY(s);
  DspgnSolver::Gather& G = s->gather;
  if (!G.active || G.rank != 0 || n > G.n_slots) return fail(DSPGN_E_ARG, "gather_results: rank 0 only, n <= n_slots");
  CU(cudaSetDevice(s->device));
  const size_t bytes = sizeof(DspgnObjectOut) * (size_t)n;
  if (G.h_out.reserve(bytes + 64)) return fail(DSPGN_E_ALLOC, "cudaMallocHost");
  CU(cudaMemcpyAsync(G.h_out.p, dspgn_gather_device(s, seq), bytes, cudaMemcpyDeviceToHost, s->stream));
  CU(cudaMemcpyAsync(G.h_out.as<unsigned char>() + bytes, G.d_local.p, 4, cudaMemcpyDeviceToHost, s->stream));
  CU(sync_stream(s));
  memcpy(out, G.h_out.p, bytes);
  int err = 0;
  memcpy(&err, G.h_out.as<unsigned char>() + bytes, 4);
  if (err) { cudaMemset(G.d_local.p, 0, 4); return fail(DSPGN_E_PEER, "a rank did not publish its results within the timeout"); }
  return 0;
}

long long dspgn_gather_wait_ns(DspgnSolver* s) {
  if (!s || !s->gather.active) return -1;
  if (s->flight.active) { fail(DSPGN_E_BUSY, "a submitted keyframe call is in flight"); return -1; }
  long long v[2] = {0, 0};
  cudaSetDevice(s->device);
  if (sync_stream(s) != cudaSuccess) return -1;
  if (cudaMemcpy(v, s->gather.d_local.p, 16, cudaMemcpyDeviceToHost) != cudaSuccess) return -1;
  return v[1];
}

__global__ void k_debug_exp(const float* x, int n, int sim3, float* out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) exp_sim3_dev(x + 7 * i, sim3 != 0, out + 12 * i);
}

int dspgn_debug_exp(int device, int sim3, const float* x, int n, float* out) {
  if (!x || !out || n < 1) return fail(DSPGN_E_ARG, "bad argument");
  CU(cudaSetDevice(device));
  DevBuf dx, dout;
  if (dx.reserve(28 * (size_t)n) || dout.reserve(48 * (size_t)n)) return fail(DSPGN_E_ALLOC, "cudaMalloc");
  CU(cudaMemcpy(dx.p, x, 28 * (size_t)n, cudaMemcpyHostToDevice));
  k_debug_exp<<<(n + 63) / 64, 64>>>(dx.as<float>(), n, sim3, dout.as<float>());
  cudaError_t e = cudaDeviceSynchronize();
  if (e == cudaSuccess) e = cudaMemcpy(out, dout.p, 48 * (size_t)n, cudaMemcpyDeviceToHost);
  dx.release(); dout.release();
  if (e != cudaSuccess) return fail(DSPGN_E_CUDA, std::string("debug_exp: ") + cudaGetErrorString(e));
  return 0;
}

const float* dspgn_results_device(DspgnSolver* s) {
  if (s && s->flight.active) { fail(DSPGN_E_BUSY, "a submitted keyframe call is in flight"); return nullptr; }
  return s ? s->d_results.as<float>() : nullptr;
}

namespace {
// The host side of a run's end, once its records and (persistent kernel) queue counters hq are on the host: the kernel's
// row totals and abort flag.
int collect_run(DspgnSolver* s, const QueueCounters* hq) {
  if (!hq) return 0;
  s->mega_ran = false;
  if (s->band_rows_pending) {                // roofline accounting: what the reference decodes (loss.py:77-78, :143-144)
    s->ctr.rows_fwd_bwd += hq->band_rows_total;                 // band rows of all iterations
    s->ctr.rows_fwd_only += (long long)hq->valid_rows_total;    // V: ray samples inside the unit sphere, all iterations
  }
  s->band_rows_pending = false;
  if (hq->abort_flag) return fail(DSPGN_E_CUDA, "persistent kernel: a work-queue wait timed out (aborted softly; results incomplete)");
  return 0;
}

// The row counters of a stopped run: the run counted every slot's rows for its full iteration count, a STOPPED slot ran
// iters_done iterations.  Slots n.. are the joint slots of gated objects; woken_added: kf_records counts theirs.
void uncount_stopped(DspgnSolver* s, const DspgnObjectOut* res, int n, int slots, bool mega, bool woken_added) {
  const DspgnConfig& c = s->cfg;
  for (int k = 0; k < slots; ++k) {
    if (res[k].status != DSPGN_ST_STOPPED || (k >= n && woken_added)) continue;
    const long long missing = c.num_iterations - res[k].iters_done;
    const ObjMeta& M = s->h_meta[k];
    s->ctr.rows_fwd_bwd -= missing * M.n_pts;
    if (!mega && !c.sdf_only) s->ctr.rows_fwd_only -= missing * M.n_rays * c.num_depth_samples;   // the kernel counts its own
  }
}
}  // namespace

int dspgn_results(DspgnSolver* s, DspgnObjectOut* out) {
  if (!s || !out) return fail(DSPGN_E_ARG, "null argument");
  BUSY(s);
  CU(cudaSetDevice(s->device));
  static_assert(sizeof(DspgnObjectOut) == 4 * DSPGN_RESULT_FLOATS, "result record layout");
  const size_t bytes = sizeof(DspgnObjectOut) * (size_t)s->n_obj;
  const bool mega = s->mega_ran;           // the queue counters (abort flag, band-row total) ride on the same copy + sync
  const size_t ctr_off = (bytes + 63) / 64 * 64;
  if (s->h_results.reserve(ctr_off + sizeof(QueueCounters))) return fail(DSPGN_E_ALLOC, "cudaMallocHost");
  const QueueCounters& hq = *reinterpret_cast<const QueueCounters*>(s->h_results.as<unsigned char>() + ctr_off);
  CU(cudaMemcpyAsync(s->h_results.p, s->d_results.p, bytes, cudaMemcpyDeviceToHost, s->stream));
  if (mega) CU(cudaMemcpyAsync(s->h_results.as<unsigned char>() + ctr_off, s->d_q_ctr.p, sizeof(QueueCounters), cudaMemcpyDeviceToHost, s->stream));
  CU(sync_stream(s));
  memcpy(out, s->h_results.p, bytes);
  return collect_run(s, mega ? &hq : nullptr);
}

namespace {
// dspgn_reconstruct_batch / dspgn_estimate_pose_batch: any number of objects in `mode`, as resident batches of at most
// kMaxObjScan one after the other, each collected before the next.  `stoppable`: the call holds a StopScope; each
// batch takes the stop hook's object if it has it, and a stopped object's rows come off the counters.
int whole_batch(DspgnSolver* s, int n_obj, const DspgnObjectIn* in, DspgnObjectOut* out, int mode, bool stoppable) {
  LinScope lin(s);
  if (int rc = lin.begin(n_obj, n_obj)) return rc;
  for (int o0 = 0; o0 < n_obj; o0 += kMaxObjScan) {
    const int n = std::min(kMaxObjScan, n_obj - o0);
    if (int rc = upload_batch_impl(s, n, in + o0, false)) return rc;
    RunArgs ra;
    if (stoppable && s->call_stop_obj >= o0 && s->call_stop_obj < o0 + n) ra.stop_slot = s->call_stop_obj - o0;
    s->lin_base = o0;
    if (int rc = run_uniform(s, mode, ra)) return rc;
    const bool mega = s->mega_ran;
    if (int rc = dspgn_results(s, out + o0)) return rc;
    if (stoppable) uncount_stopped(s, out + o0, n, n, mega, false);
    for (int k = o0; k < o0 + n; ++k)
      s->info_items[k] = info_item(s, out[k], k, mode == DSPGN_MODE_POSE ? in[k].scale : 0.f);
  }
  s->info_valid = true;
  return 0;
}
}  // namespace

int dspgn_reconstruct_batch(DspgnSolver* s, int n_obj, const DspgnObjectIn* in, DspgnObjectOut* out) {
  if (!s || !in || !out || n_obj < 1) return fail(DSPGN_E_ARG, "bad argument");
  BUSY(s);
  StopScope stop(s);
  return whole_batch(s, n_obj, in, out, DSPGN_MODE_JOINT, true);
}

int dspgn_estimate_pose_batch(DspgnSolver* s, int n_obj, const DspgnObjectIn* in, DspgnObjectOut* out) {
  if (!s || !in || !out || n_obj < 1) return fail(DSPGN_E_ARG, "bad argument");
  BUSY(s);
  for (int o = 0; o < n_obj; ++o)
    if (!in[o].code || !(in[o].scale > 0.f)) return fail(DSPGN_E_ARG, "estimate_pose needs a code and a positive scale per object");
  return whole_batch(s, n_obj, in, out, DSPGN_MODE_POSE, false);
}

namespace {

struct MeshWs {                      // one chunk's mesh workspace (mesh_count)
  uint8_t* mask; uint8_t* ok; int* vscan; int* fscan; int* bases;
  unsigned bv, bc;                   // blocks of the per-lattice-vertex / per-cube passes
};
int mesh_count(DspgnSolver* s, const MeshGrid& g, MeshWs& w);
int mesh_emit(DspgnSolver* s, const MeshGrid& g, const MeshWs& w, size_t V, size_t F);
int mesh_chunk(DspgnSolver* s, const MeshGrid& g, int32_t* nV, int32_t* nF);

// A keyframe call (dspgn_keyframe_batch_gated / _meshed / _submit) after its argument checks.  The objects are walked in
// units -- one object, or a mono pair (its two hypotheses next to each other) -- packed into resident chunks of at most
// kMaxObjScan slots; a gated object's joint slot is appended after the chunk's objects.  When meshing, a chunk also
// holds at most kMeshChunkRows grid rows of candidates, and its grids sit in walk order in the call's grid block.
struct KfWalk {
  const DspgnObjectIn* in = nullptr; const int32_t* modes = nullptr; const DspgnGateIn* gates = nullptr;
  const int32_t* pair = nullptr;
  bool mesh = false;
  int n_obj = 0, dim = 0, n_cand = 0;
  long long R = 0;                   // grid rows of one candidate
  std::vector<int> order;            // every object once, the flipped hypothesis j right after its map-pose hypothesis i < j
  std::vector<float> pose_scale;     // per object: the scale of a pose-only object, 0 for a joint one (info_item)
  bool gated(int o) const { return gates != nullptr && gates[o].gate != 0; }
  bool paired(int o) const { return pair != nullptr && pair[o] >= 0; }
  bool candidate(int o) const { return modes[o] == DSPGN_MODE_JOINT || gated(o); }
};

int kf_walk(DspgnSolver* s, int n_obj, const DspgnObjectIn* in, const int32_t* modes, const DspgnGateIn* gates,
            const DspgnMeshSpec* mesh, KfWalk& w) {
  if (!s || !in || !modes || n_obj < 1) return fail(DSPGN_E_ARG, "bad argument");
  if (int rc = check_modes(s, modes, n_obj, in)) return rc;
  w.in = in; w.modes = modes; w.gates = gates; w.n_obj = n_obj; w.mesh = mesh != nullptr;
  for (int o = 0; gates && o < n_obj; ++o) {
    const DspgnGateIn& g = gates[o];
    if (g.gate != 0 && g.gate != 1) return fail(DSPGN_E_ARG, "gate must be 0 or 1");
    if (!w.gated(o)) continue;
    if (modes[o] != DSPGN_MODE_POSE) return fail(DSPGN_E_ARG, "a gate needs a pose-only object");
    if (!g.t_cam_obj_map || !g.t_cam_obj_sim3) return fail(DSPGN_E_ARG, "a gate needs t_cam_obj_map and t_cam_obj_sim3");
    if (in[o].t_cam_world) return fail(DSPGN_E_ARG, "a gated object takes camera-frame inputs (no t_cam_world)");
  }
  w.pair = mesh ? mesh->pair : nullptr;
  w.dim = mesh ? mesh->voxels_dim : 0;
  if (mesh) {
    if (w.dim < 2 || w.dim > kMeshMaxDim) return fail(DSPGN_E_ARG, "voxels_dim must be in [2,128]");
    for (int o = 0; w.pair && o < n_obj; ++o) {
      const int j = w.pair[o];
      if (j == -1) continue;
      if (j < 0 || j >= n_obj || j == o || w.pair[j] != o) return fail(DSPGN_E_ARG, "pair must be symmetric, in range and never an object with itself");
      if (modes[o] != DSPGN_MODE_JOINT || w.gated(o)) return fail(DSPGN_E_ARG, "a pair needs two ungated joint objects");
    }
  }
  w.R = mesh ? (long long)w.dim * w.dim * w.dim : 0;
  w.order.reserve(n_obj);
  w.pose_scale.assign(n_obj, 0.f);
  for (int o = 0; o < n_obj; ++o) {
    if (modes[o] == DSPGN_MODE_POSE) w.pose_scale[o] = in[o].scale;
    w.n_cand += w.candidate(o) ? 1 : 0;
    if (w.paired(o) && w.pair[o] < o) continue;
    w.order.push_back(o);
    if (w.paired(o)) w.order.push_back(w.pair[o]);
  }
  return 0;
}

// the end of the chunk that starts at walk position u0, and its resident slots
size_t kf_chunk_end(const KfWalk& w, size_t u0, int& slots) {
  size_t u1 = u0;
  long long cands = 0;
  slots = 0;
  while (u1 < w.order.size()) {
    const int o = w.order[u1], m = w.paired(o) ? 2 : 1;
    const int sl = m + (w.gated(o) ? 1 : 0), cd = m == 2 ? 2 : (w.candidate(o) ? 1 : 0);
    if (slots + sl > kMaxObjScan || (cands + cd) * w.R > kMeshChunkRows) break;
    slots += sl; cands += cd; u1 += m;
  }
  return u1;
}

// the call's grid block and query grid; no mesh of an earlier call is returned any more
int kf_grids(DspgnSolver* s, const KfWalk& w) {
  CU(cudaSetDevice(s->device));
  s->mesh_n = 0;
  s->mesh_v.clear(); s->mesh_f.clear();
  const size_t grid_bytes = 4 * (size_t)w.n_cand * w.R;
  if (s->d_mgrid.cap < grid_bytes || s->d_grid_pts.cap < 12 * (size_t)w.R) CU(settle_stream(s));
  if (s->d_mgrid.reserve(grid_bytes) || s->d_grid_pts.reserve(12 * (size_t)w.R)) return fail(DSPGN_E_ALLOC, "grid allocation failed");
  return 0;
}

// Enqueues the chunk of walk units [u0, u0 + n) with `slots` resident slots: upload, run and, when meshing, the mesh
// selection and the decode of the chunk's grids (from grid g0 of the call).  link: per slot, as the run table has it;
// gc: grids of the chunk; grid_of[o]: the call-wide grid of each candidate object.
int kf_enqueue_chunk(DspgnSolver* s, const KfWalk& w, size_t u0, int n, int slots, int g0, bool device_wake,
                     std::vector<int32_t>& link, int& gc, std::vector<int32_t>& grid_of) {
  std::vector<DspgnObjectIn> ins;
  std::vector<int32_t> cm;
  for (int k = 0; k < n; ++k) { ins.push_back(w.in[w.order[u0 + k]]); cm.push_back(w.modes[w.order[u0 + k]]); }
  link.assign(n, -1);
  std::vector<float> t_map;
  if (slots != n) {
    t_map.assign(16 * (size_t)slots, 0.f);
    for (int k = 0; k < n; ++k) {
      const int o = w.order[u0 + k];
      if (!w.gated(o)) continue;
      const DspgnGateIn& g = w.gates[o];
      DspgnObjectIn J = w.in[o];                     // the detection as reconstruct_object(Sim3Tco, pts, rays, depth) sees it
      J.t_cam_obj = g.t_cam_obj_sim3; J.t_rs = g.sim3_rs; J.t_cs = g.sim3_cs;
      J.code = nullptr;
      link[k] = (int)ins.size();
      link.push_back(k);
      ins.push_back(J);
      cm.push_back(DSPGN_MODE_JOINT);
      for (int r = 0; r < 4; ++r)
        for (int c = 0; c < 4; ++c) t_map[16 * (size_t)k + 4 * r + c] = g.t_cam_obj_map[(size_t)r * g.map_rs + (size_t)c * g.map_cs];
    }
  }
  gc = 0;
  int* d_sel = nullptr;
  if (w.mesh) {
    // per slot: its grid in the chunk's block (-1: not a candidate) | the slot of the other hypothesis of its pair.
    // Uploaded before the run: the pairs are also the objects the call's stop leaves running.
    const size_t sel_bytes = 4 * 2 * (size_t)slots;
    if (s->d_mesh_sel.cap < sel_bytes) CU(settle_stream(s));
    if (s->d_mesh_sel.reserve(sel_bytes) || s->h_mesh_sel.reserve(sel_bytes)) return fail(DSPGN_E_ALLOC, "cudaMalloc");
    int* sel = s->h_mesh_sel.as<int>();
    std::fill(sel, sel + 2 * (size_t)slots, -1);
    for (int k = 0; k < n; ++k) {
      const int o = w.order[u0 + k];
      if (!w.candidate(o)) continue;
      sel[cm[k] == DSPGN_MODE_JOINT ? k : link[k]] = gc;
      grid_of[o] = g0 + gc++;
      if (w.paired(o)) sel[(size_t)slots + k] = w.pair[o] > o ? k + 1 : k - 1;
    }
    d_sel = s->d_mesh_sel.as<int>();
    CU(cudaMemcpyAsync(d_sel, sel, sel_bytes, cudaMemcpyHostToDevice, s->stream));
  }
  RunArgs ra;
  ra.pair = (d_sel != nullptr && w.pair != nullptr) ? d_sel + slots : nullptr;
  for (int k = 0; k < n; ++k)
    if (w.order[u0 + k] == s->call_stop_obj) ra.stop_slot = k;
  if (slots == n) {                                  // no gate in the chunk: the plain keyframe run
    if (int rc = dspgn_upload_batch(s, n, ins.data())) return rc;
    if (int rc = run_batch_impl(s, cm.data(), ra)) return rc;
  } else {
    if (int rc = dspgn_upload_batch(s, slots, ins.data())) return rc;
    if (int rc = run_batch_impl(s, cm.data(), ra, link.data(), t_map.data(), device_wake)) return rc;
  }
  if (!w.mesh) return 0;
  if (u0 == 0) {                                     // the call-wide query grid of create_voxel_grid
    k_mesh_grid_points<<<(unsigned)((w.R + 255) / 256), 256, 0, s->stream>>>(s->d_grid_pts.as<float>(), 1, w.dim);
    s->ctr.kernel_launches++;
  }
  BatchDev b = batch_dev(s, ra);
  k_mesh_select<<<slots, 128, 0, s->stream>>>(b, d_sel, d_sel + slots);
  s->ctr.kernel_launches++;
  CU(cudaGetLastError());
  if (gc > 0) {
    // grids of the candidates that get no mesh stay NaN: no cube of theirs is on the surface
    b.sdf = s->d_mgrid.as<float>() + (size_t)g0 * w.R;
    CU(cudaMemsetAsync(b.sdf, 0xff, 4 * (size_t)gc * w.R, s->stream));
    TermArgs a = base_term(s, MODE_GRIDFWD);
    a.grid = s->d_grid_pts.as<float>(); a.grid_slot = d_sel; a.grid_rows = (int)w.R;
    if (int rc = launch_term(s, b, a, (long long)gc * w.R)) return rc;
  }
  return 0;
}

// The chunk's records (res, one per slot) into the caller's out in object order; a rejected gated object gets its joint
// slot's record.  woken_rows: the woken slots' rows are not in the counters yet (1: SDF rows, 2: also ray-sample rows,
// when the run had the render term).  Each object's pose information item names the call slot (lin_base + resident
// slot) its record came from.  Returns the number of DSPGN_MESH_DONE records.
int kf_records(DspgnSolver* s, const KfWalk& w, size_t u0, int n, const std::vector<int32_t>& link,
               const DspgnObjectOut* res, DspgnObjectOut* out, int woken_rows, int lin_base) {
  int done = 0;
  for (int k = 0; k < n; ++k) {
    const int o = w.order[u0 + k];
    DspgnObjectOut& r = out[o];
    r = res[k];
    if (link[k] < 0 || res[k].gate != DSPGN_GATE_REJECTED) s->info_items[o] = info_item(s, r, lin_base + k, w.pose_scale[o]);
    if (link[k] >= 0 && res[k].gate == DSPGN_GATE_REJECTED) {
      r = res[link[k]];
      r.gate = DSPGN_GATE_REJECTED;
      s->info_items[o] = info_item(s, r, lin_base + link[k], 0.f);
      const ObjMeta& M = s->h_meta[link[k]];
      const long long iters = r.status == DSPGN_ST_STOPPED ? r.iters_done : s->cfg.num_iterations;
      if (woken_rows >= 1) s->ctr.rows_fwd_bwd += (long long)M.n_pts * iters;
      if (woken_rows >= 2) s->ctr.rows_fwd_only += (long long)M.n_rays * s->cfg.num_depth_samples * iters;
    }
    done += r.mesh == DSPGN_MESH_DONE ? 1 : 0;
  }
  return done;
}

// The call's meshes, in walk order in mesh_v / mesh_f with gV / gF per grid, into object order; the per-object counts.
void kf_meshes(DspgnSolver* s, const KfWalk& w, std::vector<int32_t>& grid_of, const std::vector<int32_t>& gV,
               const std::vector<int32_t>& gF, int32_t* n_vertices, int32_t* n_faces) {
  // they differ only where a pair is not adjacent
  bool in_order = true;
  for (int o = 0, last = -1; o < w.n_obj; ++o)
    if (grid_of[o] >= 0) { in_order = in_order && grid_of[o] > last; last = grid_of[o]; }
  if (!in_order) {
    std::vector<size_t> ov(w.n_cand + 1, 0), of(w.n_cand + 1, 0);
    for (int g = 0; g < w.n_cand; ++g) { ov[g + 1] = ov[g] + 3 * (size_t)gV[g]; of[g + 1] = of[g] + 3 * (size_t)gF[g]; }
    std::vector<float> v; std::vector<int32_t> f;
    v.reserve(s->mesh_v.size()); f.reserve(s->mesh_f.size());
    for (int o = 0; o < w.n_obj; ++o) {
      const int g = grid_of[o];
      if (g < 0) continue;
      v.insert(v.end(), s->mesh_v.begin() + ov[g], s->mesh_v.begin() + ov[g + 1]);
      f.insert(f.end(), s->mesh_f.begin() + of[g], s->mesh_f.begin() + of[g + 1]);
    }
    s->mesh_v.swap(v); s->mesh_f.swap(f);
  }
  for (int o = 0; o < w.n_obj; ++o) {
    n_vertices[o] = grid_of[o] >= 0 ? gV[grid_of[o]] : 0;
    n_faces[o] = grid_of[o] >= 0 ? gF[grid_of[o]] : 0;
  }
  s->mesh_n = w.n_obj; s->mesh_dim = w.dim;
  s->mesh_grid_of.swap(grid_of);
}

// dspgn_keyframe_batch_gated, and with mesh != nullptr dspgn_keyframe_batch_meshed: chunk after chunk, each collected
// (dspgn_results) before the next.
int keyframe_impl(DspgnSolver* s, int n_obj, const DspgnObjectIn* in, const int32_t* modes, const DspgnGateIn* gates,
                  const DspgnMeshSpec* mesh, DspgnObjectOut* out, int32_t* n_vertices, int32_t* n_faces) {
  if (!out) return fail(DSPGN_E_ARG, "bad argument");
  KfWalk w;
  if (int rc = kf_walk(s, n_obj, in, modes, gates, mesh, w)) return rc;
  BUSY(s);
  StopScope stop(s);
  LinScope lin(s);
  size_t call_slots = n_obj;                           // a gated object's joint run takes a slot of its own
  for (int o = 0; o < n_obj; ++o) call_slots += w.gated(o) ? 1 : 0;
  if (int rc = lin.begin(call_slots, n_obj)) return rc;
  std::vector<int32_t> gV, gF, grid_of(mesh ? n_obj : 0, -1);
  if (mesh) {
    if (int rc = kf_grids(s, w)) return rc;
    gV.assign(w.n_cand, 0); gF.assign(w.n_cand, 0);
  }
  std::vector<int32_t> link;
  std::vector<DspgnObjectOut> res;
  int g0 = 0;                                          // grids of the chunks before this one
  int lin_base = 0;                                    // call slots of the chunks before this one
  for (size_t u0 = 0; u0 < w.order.size();) {
    int slots = 0;
    const size_t u1 = kf_chunk_end(w, u0, slots);
    const int n = (int)(u1 - u0);
    int gc = 0;                                        // grids of this chunk
    s->lin_base = lin_base;
    if (int rc = kf_enqueue_chunk(s, w, u0, n, slots, g0, false, link, gc, grid_of)) return rc;
    const bool mega = s->mega_ran;
    res.resize(slots);
    if (int rc = dspgn_results(s, res.data())) return rc;
    uncount_stopped(s, res.data(), n, slots, mega, mega);
    const int done = kf_records(s, w, u0, n, link, res.data(), out, mega ? 1 : 0, lin_base);   // the woken slots' SDF rows
    lin_base += slots;
    if (gc > 0) {
      s->ctr.rows_fwd_only += (long long)done * w.R;
      const MeshGrid g{s->d_mgrid.as<float>() + (size_t)g0 * w.R, gc, w.dim, w.R, (long long)(w.dim - 1) * (w.dim - 1) * (w.dim - 1), 2.0 / (w.dim - 1)};
      if (int rc = mesh_chunk(s, g, gV.data() + g0, gF.data() + g0)) return rc;
    }
    g0 += gc;
    u0 = u1;
  }
  if (mesh) kf_meshes(s, w, grid_of, gV, gF, n_vertices, n_faces);
  s->info_valid = true;
  return 0;
}

}  // namespace

int dspgn_keyframe_batch(DspgnSolver* s, int n_obj, const DspgnObjectIn* in, const int32_t* modes, DspgnObjectOut* out) {
  return dspgn_keyframe_batch_gated(s, n_obj, in, modes, nullptr, out);
}

int dspgn_keyframe_batch_gated(DspgnSolver* s, int n_obj, const DspgnObjectIn* in, const int32_t* modes,
                               const DspgnGateIn* gates, DspgnObjectOut* out) {
  if (!modes) return fail(DSPGN_E_ARG, "bad argument");
  return keyframe_impl(s, n_obj, in, modes, gates, nullptr, out, nullptr, nullptr);
}

int dspgn_keyframe_batch_meshed(DspgnSolver* s, int n_obj, const DspgnObjectIn* in, const int32_t* modes,
                                const DspgnGateIn* gates, const DspgnMeshSpec* mesh, DspgnObjectOut* out,
                                int32_t* n_vertices, int32_t* n_faces) {
  if (!mesh || !n_vertices || !n_faces) return fail(DSPGN_E_ARG, "bad argument");
  std::vector<int32_t> joint;
  if (!modes && n_obj > 0) {
    joint.assign(n_obj, DSPGN_MODE_JOINT);
    modes = joint.data();
  }
  return keyframe_impl(s, n_obj, in, modes, gates, mesh, out, n_vertices, n_faces);
}

// ---- submitted keyframe calls ------------------------------------------------------------------------------------
// Submit enqueues what keyframe_impl does for one chunk, with two changes that keep the host out of the call: the
// per-iteration schedule wakes the rejected slots on the device (run_batch_impl, device_wake), and the meshes go into an
// arena sized beforehand (k_mesh_emit_*_arena) instead of buffers sized from a read-back of the counts.  Then the
// records, the queue counters, the mesh bases and the arena are copied into h_flight and ev_flight is recorded.
int dspgn_keyframe_submit(DspgnSolver* s, int n_obj, const DspgnObjectIn* in, const int32_t* modes,
                          const DspgnGateIn* gates, const DspgnMeshSpec* mesh) {
  std::vector<int32_t> joint;
  if (!modes && n_obj > 0) {
    joint.assign(n_obj, DSPGN_MODE_JOINT);
    modes = joint.data();
  }
  KfWalk w;
  if (int rc = kf_walk(s, n_obj, in, modes, gates, mesh, w)) return rc;
  BUSY(s);
  int slots = 0;
  const size_t u1 = kf_chunk_end(w, 0, slots);
  if (u1 < w.order.size())
    return fail(DSPGN_E_ARG, "a submitted keyframe must fit one resident chunk: at most 1024 slots (a gated object takes two) "
                             "and 2^24 candidate grid rows (the blocking calls take any size)");
  CU(cudaSetDevice(s->device));
  if (!s->ev_flight) CU(cudaEventCreateWithFlags(&s->ev_flight, cudaEventDisableTiming));
  StopScope stop(s);                                 // kept until the wait on success
  LinScope lin(s);
  if (int rc = lin.begin(slots, n_obj)) return rc;
  DspgnSolver::Flight& F = s->flight;
  F = DspgnSolver::Flight{};
  F.grid_of.assign(mesh ? n_obj : 0, -1);
  if (mesh)
    if (int rc = kf_grids(s, w)) return rc;
  s->mega_ran = false;
  int gc = 0;
  if (int rc = kf_enqueue_chunk(s, w, 0, (int)u1, slots, 0, true, F.link, gc, F.grid_of)) return rc;
  F.mega = s->mega_ran;
  auto al = [](size_t x) { return (x + 255) / 256 * 256; };
  F.o_ctr = al(sizeof(DspgnObjectOut) * (size_t)slots);
  F.o_base = F.o_ctr + al(sizeof(QueueCounters));
  F.o_arena = F.o_base + al(8 * ((size_t)gc + 1));
  MeshWs mw{};
  if (gc > 0) {
    F.g = MeshGrid{s->d_mgrid.as<float>(), gc, w.dim, w.R, (long long)(w.dim - 1) * (w.dim - 1) * (w.dim - 1), 2.0 / (w.dim - 1)};
    if (int rc = mesh_count(s, F.g, mw)) return rc;
    const double d2 = (double)w.dim * w.dim;
    F.cap_v = s->arena_force_v > 0 ? s->arena_force_v : gc * (long long)std::ceil(s->arena_v * d2);
    F.cap_f = s->arena_force_f > 0 ? s->arena_force_f : gc * (long long)std::ceil(s->arena_f * d2);
    const size_t arena_bytes = 12 * (size_t)(F.cap_v + F.cap_f);
    if (s->d_mout.cap < arena_bytes) CU(settle_stream(s));
    if (s->d_mout.reserve(arena_bytes)) return fail(DSPGN_E_ALLOC, "mesh arena allocation failed");
    const int* totals = mw.bases + 2 * gc;
    k_mesh_emit_verts_arena<<<mw.bv, 256, 0, s->stream>>>(F.g, mw.mask, mw.vscan, totals, F.cap_v, F.cap_f, s->d_mout.as<float>());
    k_mesh_emit_faces_arena<<<mw.bc, 256, 0, s->stream>>>(F.g, mw.mask, mw.vscan, mw.fscan, totals, F.cap_v, F.cap_f,
                                                          s->d_mout.as<float>());
    CU(cudaGetLastError());
    s->ctr.kernel_launches += 2;
    F.mask = mw.mask; F.vscan = mw.vscan; F.fscan = mw.fscan;
  }
  const size_t total = F.o_arena + 12 * (size_t)(F.cap_v + F.cap_f);
  if (s->h_flight.reserve(total)) return fail(DSPGN_E_ALLOC, "cudaMallocHost");
  unsigned char* h = s->h_flight.as<unsigned char>();
  CU(cudaMemcpyAsync(h, s->d_results.p, sizeof(DspgnObjectOut) * (size_t)slots, cudaMemcpyDeviceToHost, s->stream));
  if (F.mega) CU(cudaMemcpyAsync(h + F.o_ctr, s->d_q_ctr.p, sizeof(QueueCounters), cudaMemcpyDeviceToHost, s->stream));
  if (gc > 0) {
    CU(cudaMemcpyAsync(h + F.o_base, mw.bases, 8 * ((size_t)gc + 1), cudaMemcpyDeviceToHost, s->stream));
    CU(cudaMemcpyAsync(h + F.o_arena, s->d_mout.p, 12 * (size_t)(F.cap_v + F.cap_f), cudaMemcpyDeviceToHost, s->stream));
  }
  CU(cudaEventRecord(s->ev_flight, s->stream));
  F.mesh = mesh != nullptr;
  F.device_wake = !F.mega;
  F.render = !s->cfg.sdf_only;
  F.n_obj = n_obj; F.slots = slots; F.n = (int)u1; F.dim = w.dim; F.n_cand = w.n_cand; F.gc = gc;
  F.order.swap(w.order);
  F.pose_scale.swap(w.pose_scale);
  F.active = true;
  stop.keep = true;
  return 0;
}

int dspgn_keyframe_query(DspgnSolver* s) {
  if (!s) return fail(DSPGN_E_ARG, "null solver");
  if (!s->flight.active) return fail(DSPGN_E_ARG, "no submitted keyframe call");
  CU(cudaSetDevice(s->device));
  const cudaError_t e = cudaEventQuery(s->ev_flight);
  if (e == cudaSuccess) return 1;
  if (e == cudaErrorNotReady) return 0;
  return fail(DSPGN_E_CUDA, std::string("keyframe_query: ") + cudaGetErrorString(e));
}

int dspgn_keyframe_wait(DspgnSolver* s, DspgnObjectOut* out, int32_t* n_vertices, int32_t* n_faces) {
  if (!s || !out) return fail(DSPGN_E_ARG, "null argument");
  DspgnSolver::Flight& F = s->flight;
  if (!F.active) return fail(DSPGN_E_ARG, "no submitted keyframe call");
  if ((n_vertices == nullptr) == F.mesh || (n_faces == nullptr) == F.mesh)
    return fail(DSPGN_E_ARG, "n_vertices and n_faces must be given iff the submitted call had a mesh spec");
  F.active = false;                                  // collected from here on, whatever happens below
  struct StopEnd { DspgnSolver* s; ~StopEnd() { stop_end(s); } } stop_end_{s};   // the call's stop ends with the wait
  CU(cudaSetDevice(s->device));
  CU(settle_event(s, s->ev_flight));
  s->upload_pending = false;                         // the event follows every copy of the call
  s->run_upload_pending = false;
  const unsigned char* h = s->h_flight.as<unsigned char>();
  if (int rc = collect_run(s, F.mega ? reinterpret_cast<const QueueCounters*>(h + F.o_ctr) : nullptr)) return rc;
  uncount_stopped(s, reinterpret_cast<const DspgnObjectOut*>(h), F.n, F.slots, F.mega, true);
  KfWalk w;                                          // the walk's bookkeeping (the inputs are not read again)
  w.n_obj = F.n_obj; w.n_cand = F.n_cand; w.dim = F.dim; w.R = (long long)F.dim * F.dim * F.dim; w.mesh = F.mesh;
  w.order.swap(F.order);
  w.pose_scale.swap(F.pose_scale);
  const int done = kf_records(s, w, 0, F.n, F.link, reinterpret_cast<const DspgnObjectOut*>(h), out,
                              F.mega ? 1 : (F.render ? 2 : 1), 0);
  if (!F.mesh) { s->info_valid = true; return 0; }
  std::vector<int32_t> gV(F.n_cand, 0), gF(F.n_cand, 0);
  s->mesh_v.clear(); s->mesh_f.clear();
  if (F.gc > 0) {
    s->ctr.rows_fwd_only += (long long)done * w.R;
    const int* hb = reinterpret_cast<const int*>(h + F.o_base);
    const double d2 = (double)F.dim * F.dim;
    for (int g = 0; g < F.gc; ++g) {
      gV[g] = hb[2 * g + 2] - hb[2 * g]; gF[g] = hb[2 * g + 3] - hb[2 * g + 1];
      s->arena_v = std::max(s->arena_v, 1.25 * gV[g] / d2);     // the next calls' arena: a margin over the largest mesh
      s->arena_f = std::max(s->arena_f, 1.25 * gF[g] / d2);
    }
    const size_t V = (size_t)hb[2 * F.gc], Fc = (size_t)hb[2 * F.gc + 1];
    if ((long long)V <= F.cap_v && (long long)Fc <= F.cap_f) {
      const float* hv = reinterpret_cast<const float*>(h + F.o_arena);
      const int32_t* hf = reinterpret_cast<const int32_t*>(hv + 3 * F.cap_v);
      s->mesh_v.assign(hv, hv + 3 * V);
      s->mesh_f.assign(hf, hf + 3 * Fc);
    } else {                                         // the arena was too small: emit again at the exact size
      const MeshWs mw{F.mask, nullptr, F.vscan, F.fscan, nullptr, (unsigned)(((size_t)F.g.n * F.g.R + 255) / 256),
                      (unsigned)(((size_t)F.g.n * F.g.C + 255) / 256)};
      if (int rc = mesh_emit(s, F.g, mw, V, Fc)) return rc;
    }
  }
  kf_meshes(s, w, F.grid_of, gV, gF, n_vertices, n_faces);
  s->info_valid = true;
  return 0;
}

int dspgn_pose_information(DspgnSolver* s, int n, double* info, int32_t* info_status) {
  if (!s || !info || !info_status) return fail(DSPGN_E_ARG, "null argument");
  BUSY(s);
  if (!s->info_valid) return fail(DSPGN_E_ARG, "the solver's last call returned no records (or there was none)");
  if (n != (int)s->info_items.size()) return fail(DSPGN_E_ARG, "n must equal the object count of the solver's last call");
  CU(cudaSetDevice(s->device));
  auto al = [](size_t x) { return (x + 255) / 256 * 256; };
  const size_t o_info = al(sizeof(InfoItem) * (size_t)n), o_st = al(o_info + 36 * sizeof(double) * (size_t)n),
               total = o_st + 4 * (size_t)n;
  if (s->h_info.reserve(total) || s->d_info.reserve(total)) return fail(DSPGN_E_ALLOC, "pose information allocation failed");
  unsigned char* h = s->h_info.as<unsigned char>();
  unsigned char* d = s->d_info.as<unsigned char>();
  memcpy(h, s->info_items.data(), sizeof(InfoItem) * (size_t)n);
  CU(cudaMemcpyAsync(d, h, sizeof(InfoItem) * (size_t)n, cudaMemcpyHostToDevice, s->stream));
  k_pose_information<<<n, kInfoThreads, 0, s->stream>>>(s->d_lin.as<float>(), lin_floats(s->cfg.code_len),
                                                         reinterpret_cast<const InfoItem*>(d), reinterpret_cast<double*>(d + o_info),
                                                         reinterpret_cast<int*>(d + o_st));
  CU(cudaGetLastError());
  CU(cudaMemcpyAsync(h + o_info, d + o_info, total - o_info, cudaMemcpyDeviceToHost, s->stream));
  CU(sync_stream(s));
  memcpy(info, h + o_info, 36 * sizeof(double) * (size_t)n);
  memcpy(info_status, h + o_st, 4 * (size_t)n);
  return 0;
}

int dspgn_debug_host_syncs(DspgnSolver* s, int64_t* out) {
  if (!s || !out) return fail(DSPGN_E_ARG, "null argument");
  *out = s->host_syncs;
  return 0;
}

int dspgn_keyframe_stop(DspgnSolver* s) {
  if (!s) return fail(DSPGN_E_ARG, "null solver");
  request_stop(s);
  return 0;
}

int dspgn_solver_set_stop_flag(DspgnSolver* s, const volatile uint8_t* flag) {
  if (!s) return fail(DSPGN_E_ARG, "null solver");
  BUSY(s);
  s->stop_flag = flag;
  return 0;
}

int dspgn_debug_stop_at(DspgnSolver* s, int obj, int iter) {
  if (!s) return fail(DSPGN_E_ARG, "null solver");
  const int max_iter = std::max(s->cfg.num_iterations, s->cfg.pose_only_iterations);
  if (!(obj == -1 && iter == -1) && (obj < 0 || iter < 0 || iter >= max_iter))
    return fail(DSPGN_E_ARG, "stop_at: obj >= 0 and 0 <= iter < the solver's iteration count, or -1, -1");
  BUSY(s);
  s->stop_at_obj = obj; s->stop_at_iter = iter;
  return 0;
}

int dspgn_debug_mesh_arena(DspgnSolver* s, int64_t max_vertices, int64_t max_faces) {
  if (!s || max_vertices < 0 || max_faces < 0 || (max_vertices == 0) != (max_faces == 0)) return fail(DSPGN_E_ARG, "bad argument");
  BUSY(s);
  s->arena_force_v = max_vertices; s->arena_force_f = max_faces;
  return 0;
}

int dspgn_debug_sm_budget(DspgnSolver* s, int n, int32_t* current) {
  if (!s || n < 0) return fail(DSPGN_E_ARG, "bad argument");
  BUSY(s);
  if (n > s->num_sms) return fail(DSPGN_E_ARG, "n must be 0 (automatic) or in [1, number of SMs]");
  s->sm_force = n;
  if (current) *current = grid_sms(s);
  return 0;
}

namespace {
// The forward decode of the `rows` points of a resident batch uploaded decode_only, into sdf
int decode_points(DspgnSolver* s, float* sdf, long long rows) {
  const std::vector<int32_t> joint(s->n_obj, DSPGN_MODE_JOINT);
  RunPlan p;
  if (int rc = plan_run(s, joint.data(), p)) return rc;
  BatchDev b = batch_dev(s, RunArgs{});
  b.sdf = sdf;
  if (int rc = launch_init(s, b, p)) return rc;
  if (int rc = launch_term(s, b, base_term(s, MODE_PTSFWD), rows)) return rc;
  s->ctr.rows_fwd_only += rows;
  return 0;
}
}  // namespace

int dspgn_decode_sdf(DspgnSolver* s, int class_id, const float* code, const float* x, int n, int x_rs, int x_cs,
                     float* sdf_out) {
  if (!s || !code || !x || !sdf_out || n < 1) return fail(DSPGN_E_ARG, "bad argument");
  BUSY(s);
  const float I4[16] = {1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1};
  DspgnObjectIn in{};
  in.t_cam_obj = I4; in.t_rs = 4; in.t_cs = 1;
  in.pts = x; in.n_pts = n; in.pts_rs = x_rs; in.pts_cs = x_cs;
  in.rays = nullptr; in.n_rays = 0; in.depth = nullptr; in.n_depth = 0;
  in.code = code; in.scale = 1.f; in.class_id = class_id;
  if (int rc = upload_batch_impl(s, 1, &in, true)) return rc;      // forward only: no J^T J partial / band buffers
  if (s->d_sdf.reserve(4 * (size_t)n)) return fail(DSPGN_E_ALLOC, "cudaMalloc");
  if (int rc = run_begin(s)) return rc;
  if (int rc = decode_points(s, s->d_sdf.as<float>(), n)) return rc;
  if (int rc = run_end(s)) return rc;
  CU(cudaMemcpyAsync(sdf_out, s->d_sdf.p, 4 * (size_t)n, cudaMemcpyDeviceToHost, s->stream));
  CU(sync_stream(s));
  return 0;
}

namespace {

// The passes of the iso-surface of the chunk's grids g (dspgn_mesh.cuh) up to the per-object bases (w.bases: first vertex
// and face of every object, entry g.n the totals), enqueued.
int mesh_count(DspgnSolver* s, const MeshGrid& g, MeshWs& ws) {
  const size_t nv = (size_t)g.n * g.R, nf = 4 * (size_t)g.n * g.C;
  auto al = [](size_t x) { return (x + 255) / 256 * 256; };
  // workspace: vertex counts -> scan [nv + 1] | face counts -> scan [nf + 1] | edge masks [nv] | cube flags [n C] |
  // per-object bases [n + 1][2]
  const size_t o_fc = al(4 * (nv + 1)), o_mask = o_fc + al(4 * (nf + 1)), o_ok = o_mask + al(nv),
               o_base = o_ok + al((size_t)g.n * g.C), total = o_base + al(8 * ((size_t)g.n + 1));
  if (s->d_mws.cap < total) CU(settle_stream(s));
  if (s->d_mws.reserve(total)) return fail(DSPGN_E_ALLOC, "mesh workspace allocation failed");
  unsigned char* w = s->d_mws.as<unsigned char>();
  int* vscan = reinterpret_cast<int*>(w);
  int* fscan = reinterpret_cast<int*>(w + o_fc);
  uint8_t* mask = w + o_mask;
  uint8_t* ok = w + o_ok;
  int* bases = reinterpret_cast<int*>(w + o_base);
  size_t tmp_v = 0, tmp_f = 0;
  CU(cub::DeviceScan::ExclusiveSum(nullptr, tmp_v, vscan, vscan, (int)(nv + 1), s->stream));
  CU(cub::DeviceScan::ExclusiveSum(nullptr, tmp_f, fscan, fscan, (int)(nf + 1), s->stream));
  if (s->d_mscan_tmp.cap < std::max(tmp_v, tmp_f)) CU(settle_stream(s));
  if (s->d_mscan_tmp.reserve(std::max(tmp_v, tmp_f))) return fail(DSPGN_E_ALLOC, "mesh workspace allocation failed");
  // the slot after the last count: the scans' totals
  CU(cudaMemsetAsync(vscan + nv, 0, 4, s->stream));
  CU(cudaMemsetAsync(fscan + nf, 0, 4, s->stream));
  const unsigned bc = (unsigned)(((size_t)g.n * g.C + 255) / 256), bv = (unsigned)((nv + 255) / 256);
  k_mesh_cubes<<<bc, 256, 0, s->stream>>>(g, ok, fscan);
  k_mesh_verts<<<bv, 256, 0, s->stream>>>(g, ok, mask, vscan);
  CU(cudaGetLastError());
  size_t tb = s->d_mscan_tmp.cap;
  CU(cub::DeviceScan::ExclusiveSum(s->d_mscan_tmp.p, tb, vscan, vscan, (int)(nv + 1), s->stream));
  tb = s->d_mscan_tmp.cap;
  CU(cub::DeviceScan::ExclusiveSum(s->d_mscan_tmp.p, tb, fscan, fscan, (int)(nf + 1), s->stream));
  // per object: first vertex and first face (object n: the totals)
  k_mesh_bases<<<(g.n + 1 + 127) / 128, 128, 0, s->stream>>>(g, vscan, fscan, bases);
  CU(cudaGetLastError());
  s->ctr.kernel_launches += 2 + 2 * 2 + 1;                    // classify passes, two scans (two kernels each), bases
  ws = MeshWs{mask, ok, vscan, fscan, bases, bv, bc};
  return 0;
}

// The emit passes of mesh_count's chunk at V vertices and F faces, appended to s->mesh_v / mesh_f (synchronous).
int mesh_emit(DspgnSolver* s, const MeshGrid& g, const MeshWs& w, size_t V, size_t F) {
  if (V == 0 && F == 0) return 0;
  if (s->d_mout.reserve(12 * (V + F))) return fail(DSPGN_E_ALLOC, "mesh output allocation failed");
  float* dv = s->d_mout.as<float>();
  int32_t* df = reinterpret_cast<int32_t*>(dv + 3 * V);
  k_mesh_emit_verts<<<w.bv, 256, 0, s->stream>>>(g, w.mask, w.vscan, dv);
  k_mesh_emit_faces<<<w.bc, 256, 0, s->stream>>>(g, w.mask, w.vscan, w.fscan, df);
  CU(cudaGetLastError());
  s->ctr.kernel_launches += 2;
  const size_t v0 = s->mesh_v.size(), f0 = s->mesh_f.size();
  s->mesh_v.resize(v0 + 3 * V);
  s->mesh_f.resize(f0 + 3 * F);
  CU(cudaMemcpyAsync(s->mesh_v.data() + v0, dv, 12 * V, cudaMemcpyDeviceToHost, s->stream));
  CU(cudaMemcpyAsync(s->mesh_f.data() + f0, df, 12 * F, cudaMemcpyDeviceToHost, s->stream));
  CU(sync_stream(s));
  return 0;
}

// The iso-surface of the chunk's grids g, appended to s->mesh_v / mesh_f; per-object counts into nV / nF (one read-back).
int mesh_chunk(DspgnSolver* s, const MeshGrid& g, int32_t* nV, int32_t* nF) {
  MeshWs w;
  if (int rc = mesh_count(s, g, w)) return rc;
  if (s->h_mbase.reserve(8 * ((size_t)g.n + 1))) return fail(DSPGN_E_ALLOC, "mesh workspace allocation failed");
  int* hb = s->h_mbase.as<int>();
  CU(cudaMemcpyAsync(hb, w.bases, 8 * ((size_t)g.n + 1), cudaMemcpyDeviceToHost, s->stream));
  CU(sync_stream(s));
  for (int o = 0; o < g.n; ++o) { nV[o] = hb[2 * o + 2] - hb[2 * o]; nF[o] = hb[2 * o + 3] - hb[2 * o + 1]; }
  return mesh_emit(s, g, w, (size_t)hb[2 * g.n], (size_t)hb[2 * g.n + 1]);
}

// One mesh call: grids decoded from codes (sdf_in == nullptr) or given by the caller, meshed chunk after chunk.  The
// grids of the whole call stay in HBM for dspgn_mesh_results (4 B per grid row); the rest of the device memory is per
// chunk of at most kMeshChunkRows grid rows, about 34 B per row (query points 12, vertex scan 4, face scans 16, flags 2),
// plus the chunk's meshes.
int mesh_impl(DspgnSolver* s, int n, int dim, const float* codes, int code_stride, const int32_t* class_ids,
              const float* sdf_in, int32_t* n_vertices, int32_t* n_faces) {
  if (!s || n < 1 || !n_vertices || !n_faces) return fail(DSPGN_E_ARG, "bad argument");
  if (dim < 2 || dim > kMeshMaxDim) return fail(DSPGN_E_ARG, "voxels_dim must be in [2,128]");
  if (!codes && !sdf_in) return fail(DSPGN_E_ARG, "null codes");
  if (codes && code_stride < s->cfg.code_len) return fail(DSPGN_E_ARG, "code_stride must be >= code_len");
  for (int o = 0; class_ids && o < n; ++o)
    if (class_ids[o] < 0 || class_ids[o] >= (int)s->classes.size()) return fail(DSPGN_E_ARG, "bad class_id");
  BUSY(s);
  CU(cudaSetDevice(s->device));
  const long long R = (long long)dim * dim * dim, C = (long long)(dim - 1) * (dim - 1) * (dim - 1);
  const int per_chunk = (int)std::max<long long>(1, std::min<long long>(kMaxObjScan, kMeshChunkRows / R));
  s->mesh_n = 0;
  s->mesh_v.clear(); s->mesh_f.clear(); s->mesh_grid_of.clear();
  if (s->d_mgrid.cap < 4 * (size_t)n * R) CU(settle_stream(s));
  if (s->d_mgrid.reserve(4 * (size_t)n * R)) return fail(DSPGN_E_ALLOC, "grid allocation failed");
  if (int rc = run_begin(s)) return rc;
  if (sdf_in) CU(cudaMemcpyAsync(s->d_mgrid.p, sdf_in, 4 * (size_t)n * R, cudaMemcpyHostToDevice, s->stream));
  const float I4[16] = {1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1};
  std::vector<DspgnObjectIn> ins;
  for (int o0 = 0; o0 < n; o0 += per_chunk) {
    const int nc = std::min(per_chunk, n - o0);
    float* grid = s->d_mgrid.as<float>() + (size_t)o0 * R;
    if (codes) {            // dspgn_decode_sdf of the query grid, every object of the chunk in one launch
      ins.assign(nc, DspgnObjectIn{});
      for (int k = 0; k < nc; ++k) {
        DspgnObjectIn& I = ins[k];
        I.t_cam_obj = I4; I.t_rs = 4; I.t_cs = 1;
        I.n_pts = (int)R;
        I.code = codes + (size_t)(o0 + k) * code_stride; I.scale = 1.f; I.class_id = class_ids ? class_ids[o0 + k] : 0;
      }
      if (int rc = upload_batch_impl(s, nc, ins.data(), true, dim)) return rc;
      if (int rc = decode_points(s, grid, (long long)nc * R)) return rc;
    }
    const MeshGrid g{grid, nc, dim, R, C, 2.0 / (dim - 1)};
    if (int rc = mesh_chunk(s, g, n_vertices + o0, n_faces + o0)) return rc;
  }
  if (int rc = run_end(s)) return rc;
  CU(sync_stream(s));
  s->mesh_n = n; s->mesh_dim = dim;
  return 0;
}

}  // namespace

int dspgn_mesh_batch(DspgnSolver* s, int n, const float* codes, int code_stride, const int32_t* class_ids,
                     int voxels_dim, int32_t* n_vertices, int32_t* n_faces) {
  if (!codes) return fail(DSPGN_E_ARG, "null codes");
  return mesh_impl(s, n, voxels_dim, codes, code_stride, class_ids, nullptr, n_vertices, n_faces);
}

int dspgn_debug_mesh_grid(DspgnSolver* s, int n, int voxels_dim, const float* sdf, int32_t* n_vertices, int32_t* n_faces) {
  if (!sdf) return fail(DSPGN_E_ARG, "null sdf");
  return mesh_impl(s, n, voxels_dim, nullptr, 0, nullptr, sdf, n_vertices, n_faces);
}

int dspgn_mesh_results(DspgnSolver* s, float* vertices, int32_t* faces, float* sdf) {
  if (!s) return fail(DSPGN_E_ARG, "null solver");
  BUSY(s);
  if (s->mesh_n < 1) return fail(DSPGN_E_ARG, "no mesh call to return");
  if ((!vertices && !s->mesh_v.empty()) || (!faces && !s->mesh_f.empty())) return fail(DSPGN_E_ARG, "null output");
  if (!s->mesh_v.empty()) memcpy(vertices, s->mesh_v.data(), 4 * s->mesh_v.size());
  if (!s->mesh_f.empty()) memcpy(faces, s->mesh_f.data(), 4 * s->mesh_f.size());
  if (sdf) {
    CU(cudaSetDevice(s->device));
    const size_t R = (size_t)s->mesh_dim * s->mesh_dim * s->mesh_dim;
    if (s->mesh_grid_of.empty()) {
      CU(cudaMemcpyAsync(sdf, s->d_mgrid.p, 4 * (size_t)s->mesh_n * R, cudaMemcpyDeviceToHost, s->stream));
    } else {
      for (int o = 0; o < s->mesh_n; ++o) {
        const int g = s->mesh_grid_of[o];
        if (g >= 0) CU(cudaMemcpyAsync(sdf + (size_t)o * R, s->d_mgrid.as<float>() + (size_t)g * R, 4 * R, cudaMemcpyDeviceToHost, s->stream));
        else memset(sdf + (size_t)o * R, 0xff, 4 * R);     // no grid: NaN, the bit pattern of the device's unmeshed grids
      }
    }
    CU(sync_stream(s));
  }
  return 0;
}

int dspgn_debug_system(DspgnSolver* s, int obj, int mode, float* H, float* b, float* dx, float* J_rows,
                       float* res_rows, float* losses) {
  return dspgn_debug_system_iter(s, obj, mode, 0, H, b, dx, J_rows, res_rows, losses);
}

int dspgn_debug_system_iter(DspgnSolver* s, int obj, int mode, int iter, float* H, float* b, float* dx, float* J_rows,
                            float* res_rows, float* losses) {
  if (!s || !H || !b || !dx) return fail(DSPGN_E_ARG, "null argument");
  BUSY(s);
  if (obj < 0 || obj >= s->n_obj) return fail(DSPGN_E_ARG, "bad object index");
  if (iter < 0 || iter > 1000) return fail(DSPGN_E_ARG, "bad iteration index");
  if (mode != DSPGN_MODE_JOINT && mode != DSPGN_MODE_POSE) return fail(DSPGN_E_ARG, "mode must be 0 or 1");
  CU(cudaSetDevice(s->device));
  const std::vector<int32_t> modes(s->n_obj, mode);
  RunPlan p;
  if (int rc = plan_run(s, modes.data(), p, true)) return rc;
  const int P = (mode == DSPGN_MODE_POSE) ? 6 : 7 + s->cfg.code_len;
  const int npts = s->h_meta[obj].n_pts;
  DevBuf dJ;
  if (dJ.reserve(4 * ((size_t)npts * P + npts))) return fail(DSPGN_E_ALLOC, "cudaMalloc");
  float* dJp = dJ.as<float>();
  float* dres = dJp + (size_t)npts * P;
  const BatchDev bd = batch_dev(s, RunArgs{});
  int rc = run_begin(s);
  if (!rc) rc = launch_init(s, bd, p);
  if (!rc) rc = gn_iterations(s, bd, p, iter);       // advance the whole batch `iter` GN iterations (per-iteration schedule)
  if (!rc) rc = launch_terms(s, bd, p, iter, dJp, dres, obj, P);
  if (!rc) {
    SolveArgs v = base_solve(s);
    float* d = s->d_dbg.as<float>();
    v.dbg_obj = obj; v.dbg_H = d; v.dbg_b = d + kPMax * kPMax; v.dbg_dx = v.dbg_b + kPMax; v.dbg_loss = v.dbg_dx + kPMax;
    v.iter_index = iter;
    cudaMemsetAsync(d, 0, 4 * ((size_t)kPMax * kPMax + 2 * kPMax + 8), s->stream);
    rc = launch_solve(s, bd, v);
    if (!rc) rc = run_end(s);
    if (!rc) {
      cudaMemcpyAsync(H, v.dbg_H, 4 * (size_t)P * P, cudaMemcpyDeviceToHost, s->stream);
      cudaMemcpyAsync(b, v.dbg_b, 4 * (size_t)P, cudaMemcpyDeviceToHost, s->stream);
      cudaMemcpyAsync(dx, v.dbg_dx, 4 * (size_t)P, cudaMemcpyDeviceToHost, s->stream);
      if (losses) cudaMemcpyAsync(losses, v.dbg_loss, 16, cudaMemcpyDeviceToHost, s->stream);
      if (J_rows) cudaMemcpyAsync(J_rows, dJp, 4 * (size_t)npts * P, cudaMemcpyDeviceToHost, s->stream);
      if (res_rows) cudaMemcpyAsync(res_rows, dres, 4 * (size_t)npts, cudaMemcpyDeviceToHost, s->stream);
    }
  }
  cudaError_t e = sync_stream(s);
  dJ.release();
  if (rc) return rc;
  if (e != cudaSuccess) return fail(DSPGN_E_CUDA, std::string("debug_system: ") + cudaGetErrorString(e));
  return 0;
}

int dspgn_debug_inputs(DspgnSolver* s, int obj, float* t_cam_obj, float* pts, float* rays) {
  if (!s || obj < 0 || obj >= s->n_obj) return fail(DSPGN_E_ARG, "bad argument");
  BUSY(s);
  CU(cudaSetDevice(s->device));
  CU(sync_stream(s));
  const ObjMeta& M = s->h_meta[obj];
  if (t_cam_obj) CU(cudaMemcpy(t_cam_obj, s->d_Tinit + 16 * (size_t)obj, 64, cudaMemcpyDeviceToHost));
  if (pts && M.n_pts) CU(cudaMemcpy(pts, s->d_pts + 3 * (size_t)M.pts_off, 12 * (size_t)M.n_pts, cudaMemcpyDeviceToHost));
  if (rays && M.n_rays) CU(cudaMemcpy(rays, s->d_rays + 3 * (size_t)M.ray_off, 12 * (size_t)M.n_rays, cudaMemcpyDeviceToHost));
  return 0;
}

int dspgn_debug_events(DspgnSolver* s, long long* out, int max_events) {
  // event log of the last persistent-kernel run (env DSPGN_CLK=1 at solver creation): returns the number of events,
  // out[2*i] = %globaltimer (ns), out[2*i+1] = kind<<56 | mode<<52 | sm<<40 | object<<24 | tile (or iteration)
  if (!s || !out || max_events < 1) return fail(DSPGN_E_ARG, "bad argument");
  BUSY(s);
  if (!s->events_on || !s->d_ev.p) return fail(DSPGN_E_ARG, "event log not enabled (DSPGN_CLK)");
  CU(cudaSetDevice(s->device));
  CU(sync_stream(s));
  long long n = 0;
  CU(cudaMemcpy(&n, s->d_ev.p, 8, cudaMemcpyDeviceToHost));
  if (n > kEvCap) n = kEvCap;
  if (n > max_events) n = max_events;
  CU(cudaMemcpy(out, s->d_ev.as<long long>() + 1, 16 * (size_t)n, cudaMemcpyDeviceToHost));
  return (int)n;
}

int dspgn_tc_selftest(int device, int n_mma, int k_steps, const float* A, const float* B, float* D) {
  // D[128][n_mma] = A[128][16*k_steps] * B[n_mma][16*k_steps]^T through the tensor-core operand paths
  if (!A || !B || !D || n_mma < 16 || n_mma > 256 || (n_mma % 16) || k_steps < 1 || k_steps > 16) return fail(DSPGN_E_ARG, "bad selftest shape");
  CU(cudaSetDevice(device));
  if (int rc = tc_setup_kernels(g_err)) return rc;
  const int K = 16 * k_steps;
  std::vector<unsigned char> blob;
  tc_pack_images(blob, tc_mma_n(n_mma), tc_pad_k_steps(k_steps),
                 [&](int n, int kk) { return (n < n_mma && kk < K) ? B[(size_t)n * K + kk] : 0.f; });
  DevBuf dA, dB, dD;
  if (dA.reserve(4 * (size_t)128 * K) || dB.reserve(blob.size()) || dD.reserve(4 * (size_t)128 * n_mma)) return fail(DSPGN_E_ALLOC, "cudaMalloc");
  CU(cudaMemcpy(dA.p, A, 4 * (size_t)128 * K, cudaMemcpyHostToDevice));
  CU(cudaMemcpy(dB.p, blob.data(), blob.size(), cudaMemcpyHostToDevice));
  k_tc_selftest<<<1, kTcThreads, kTcSelftestSmem>>>(dA.as<float>(), K, dB.as<unsigned char>(), n_mma, k_steps, dD.as<float>());
  cudaError_t e = cudaDeviceSynchronize();
  if (e == cudaSuccess) e = cudaMemcpy(D, dD.p, 4 * (size_t)128 * n_mma, cudaMemcpyDeviceToHost);
  dA.release(); dB.release(); dD.release();
  if (e != cudaSuccess) return fail(DSPGN_E_CUDA, std::string("tc_selftest: ") + cudaGetErrorString(e));
  return 0;
}

#ifdef DSPGN_STALL_PROBE
// probe build only (tools/tile_probe.py): copies the per-CTA cycle counters of the tensor-core tile loop into out
// (kProbeCtas x 3 x kProbeSlots), then zeroes them when `reset`.  Returns the number of values.
int dspgn_debug_stall_probe(int device, unsigned long long* out, int reset) {
  CU(cudaSetDevice(device));
  CU(cudaDeviceSynchronize());
  constexpr size_t n = (size_t)kProbeCtas * 3 * kProbeSlots;
  if (out) CU(cudaMemcpyFromSymbol(out, g_stall_probe, 8 * n));
  if (reset) {
    std::vector<unsigned long long> zero(n, 0ull);
    CU(cudaMemcpyToSymbol(g_stall_probe, zero.data(), 8 * n));
  }
  return (int)n;
}
#endif

}  // extern "C"

// ---- frame handles: what DspgnLidarFrame and DspgnMonoFrame share ----

namespace {

struct FrameCore {
  int device = 0;
  cudaStream_t stream = nullptr;
  cudaStream_t own = nullptr;  // the handle's non-blocking stream (the default), so LocalMapping's work never orders it
  HostBuf h_in, h_out;        // pinned: staged inputs, downloaded outputs
  DevBuf d_in, d_work, d_out;
};

size_t align16(size_t x) { return (x + 15) & ~(size_t)15; }

// A frame handle's own stream: non-blocking, at the device's greatest priority, so that the frame's blocks are
// dispatched ahead of the solver's queued short kernels (mesh passes, scans, per-iteration launches).
int frame_stream(cudaStream_t* out) {
  int least = 0, greatest = 0;
  if (cudaDeviceGetStreamPriorityRange(&least, &greatest) != cudaSuccess ||
      cudaStreamCreateWithPriority(out, cudaStreamNonBlocking, greatest) != cudaSuccess) {
    cudaGetLastError();
    return fail(DSPGN_E_CUDA, "cudaStreamCreateWithPriority");
  }
  return 0;
}

// A new handle on its own stream, counted as a live frame of the device (grid_sms) until frame_destroy
template <class F, class Spec>
int frame_create(const Spec& spec, int device, F** out) {
  if (int rc = check_device(device)) return rc;
  F* f = new (std::nothrow) F();
  if (!f) return fail(DSPGN_E_ALLOC, "oom");
  f->device = device;
  f->spec = spec;
  if (int rc = frame_stream(&f->own)) {
    delete f;
    return rc;
  }
  f->stream = f->own;
  count_frame(device, 1);
  *out = f;
  return 0;
}

template <class F>
void frame_destroy(F* f) {
  if (!f) return;
  cudaSetDevice(f->device);
  cudaStreamSynchronize(f->stream);
  f->h_in.release(); f->h_out.release();
  f->d_in.release(); f->d_work.release(); f->d_out.release();
  if (f->own) cudaStreamDestroy(f->own);
  count_frame(f->device, -1);
  delete f;
}

int frame_set_stream(FrameCore* f, void* cuda_stream) {
  if (!f) return fail(DSPGN_E_ARG, "null frame");
  f->stream = reinterpret_cast<cudaStream_t>(cuda_stream);
  return 0;
}

// every mask's box (l, t, r, b) inside the image
int check_bboxes(const int32_t* bboxes, int n_masks, int img_w, int img_h) {
  for (int m = 0; m < n_masks; ++m) {
    const int32_t* bb = bboxes + 4 * m;
    if (!(0 <= bb[0] && bb[0] <= bb[2] && bb[2] <= img_w && 0 <= bb[1] && bb[1] <= bb[3] && bb[3] <= img_h))
      return fail(DSPGN_E_ARG, "bbox " + std::to_string(m) + " outside 0 <= l <= r <= img_w, 0 <= t <= b <= img_h");
  }
  return 0;
}

// the masks of img_h x img_w bytes each into the staging block at dst, each padded with zeros to mstride bytes
void stage_masks(unsigned char* dst, const uint8_t* masks, int n_masks, size_t hw, size_t mstride) {
  for (int m = 0; m < n_masks; ++m) {
    memcpy(dst + m * mstride, masks + m * hw, hw);
    memset(dst + m * mstride + hw, 0, mstride - hw);
  }
}

}  // namespace

// ---- LiDAR keyframe detections (dspgn_frame.cuh) ----

struct DspgnLidarFrame : FrameCore {
  DspgnLidarSpec spec{};
  int n_boxes = 0;            // of the last run
  std::vector<DspgnLidarBoxOut> last;
};

namespace {

// the output block of a run: header, points [box][num_max][3], rays [box][num_max + 200][3]
struct FrameOutLayout {
  size_t hdr, pts, rays, bytes;
  FrameOutLayout(int n_boxes, int num_max) {
    hdr = 0;
    pts = align16(4 * (size_t)n_boxes * kFrameHdr);
    rays = pts + align16(12 * (size_t)n_boxes * num_max);
    bytes = rays + 12 * (size_t)n_boxes * (num_max + kFrameBackground);
  }
};

}  // namespace

extern "C" {

int dspgn_lidar_frame_create(const DspgnLidarSpec* spec, int device, DspgnLidarFrame** out) {
  if (!spec || !out) return fail(DSPGN_E_ARG, "null argument");
  if (spec->img_h < 1 || spec->img_h > 4096 || spec->img_w < 1 || spec->img_w > 4096) return fail(DSPGN_E_ARG, "image size must be in [1,4096]^2");
  if (spec->num_lidar_max < 1 || spec->num_lidar_max > kFrameMaxLidar) return fail(DSPGN_E_ARG, "num_lidar_max must be in [1,4096]");
  if (spec->downsample_ratio < 1) return fail(DSPGN_E_ARG, "downsample_ratio must be >= 1");
  return frame_create(*spec, device, out);
}

void dspgn_lidar_frame_destroy(DspgnLidarFrame* f) { frame_destroy(f); }

int dspgn_lidar_frame_set_stream(DspgnLidarFrame* f, void* cuda_stream) { return frame_set_stream(f, cuda_stream); }

int dspgn_lidar_frame_run(DspgnLidarFrame* f, const float* scan, int n_points, const DspgnLidarBox* boxes, int n_boxes,
                          const uint8_t* masks, const int32_t* bboxes, int n_masks, DspgnLidarBoxOut* out) {
  if (!f) return fail(DSPGN_E_ARG, "null frame");
  const DspgnLidarSpec& sp = f->spec;
  if (n_points < 0 || n_points > (1 << 22)) return fail(DSPGN_E_ARG, "n_points must be in [0, 2^22]");
  if (n_boxes < 0 || n_boxes > kFrameMaxBoxes) return fail(DSPGN_E_ARG, "n_boxes must be in [0, 256]");
  if (n_masks < 0 || n_masks > kFrameMaxMasks) return fail(DSPGN_E_ARG, "n_masks must be in [0, 64]");
  if ((n_points > 0 && !scan) || (n_boxes > 0 && (!boxes || !out)) || (n_masks > 0 && (!masks || !bboxes)))
    return fail(DSPGN_E_ARG, "null pointer where data is required");
  if (int rc = check_bboxes(bboxes, n_masks, sp.img_w, sp.img_h)) return rc;
  CU(cudaSetDevice(f->device));
  f->n_boxes = n_boxes;
  f->last.assign(n_boxes, DspgnLidarBoxOut{0, -1, -1, 0});
  if (n_boxes == 0) return 0;
  // staged input block: boxes | bboxes | scan | masks (each mask padded to 16 bytes)
  const size_t mstride = align16((size_t)sp.img_h * sp.img_w);
  const size_t o_bb = align16(4 * (size_t)n_boxes * kFrameBoxWords);
  const size_t o_scan = o_bb + align16(16 * (size_t)n_masks);
  const size_t o_mask = o_scan + align16(16 * (size_t)n_points);
  const size_t in_bytes = o_mask + mstride * n_masks;
  const int n_chunks = (n_points + kFrameChunk - 1) / kFrameChunk;
  const size_t o_tot = align16(4 * (size_t)n_boxes * std::max(n_chunks, 1));
  const size_t o_area = o_tot + align16(4 * (size_t)n_boxes);
  const size_t work_bytes = o_area + 4 * (size_t)kFrameMaxMasks;
  const FrameOutLayout L(n_boxes, sp.num_lidar_max);
  if (f->h_in.reserve(in_bytes) || f->h_out.reserve(L.bytes)) return fail(DSPGN_E_ALLOC, "cudaMallocHost");
  if (f->d_in.reserve(in_bytes) || f->d_work.reserve(work_bytes) || f->d_out.reserve(L.bytes)) return fail(DSPGN_E_ALLOC, "cudaMalloc");
  unsigned char* h = f->h_in.as<unsigned char>();
  float* hb = reinterpret_cast<float*>(h);
  for (int b = 0; b < n_boxes; ++b) {
    float* w = hb + (size_t)b * kFrameBoxWords;
    memcpy(w, boxes[b].t_obj_velo, 12 * sizeof(float));
    memcpy(w + 12, boxes[b].trans, 3 * sizeof(float));
    memcpy(w + 15, boxes[b].size, 3 * sizeof(float));
    const int32_t front = boxes[b].front != 0;
    memcpy(w + 18, &front, 4);
    w[19] = 0.f;
  }
  if (n_masks) memcpy(h + o_bb, bboxes, 16 * (size_t)n_masks);
  if (n_points) memcpy(h + o_scan, scan, 16 * (size_t)n_points);
  stage_masks(h + o_mask, masks, n_masks, (size_t)sp.img_h * sp.img_w, mstride);
  FrameParams P{};
  memcpy(P.K, sp.k, sizeof(P.K));
  memcpy(P.inv_k, sp.inv_k, sizeof(P.inv_k));
  memcpy(P.tcv, sp.t_cam_velo, sizeof(P.tcv));
  P.img_h = sp.img_h; P.img_w = sp.img_w; P.num_max = sp.num_lidar_max; P.min_area = sp.min_mask_area;
  P.alpha = sp.downsample_ratio; P.n_pts = n_points; P.n_boxes = n_boxes; P.n_masks = n_masks; P.n_chunks = n_chunks;
  P.mask_stride = (long long)mstride;
  unsigned char* d = f->d_in.as<unsigned char>();
  const float* d_boxes = reinterpret_cast<const float*>(d);
  const int* d_bb = reinterpret_cast<const int*>(d + o_bb);
  const float4* d_scan = reinterpret_cast<const float4*>(d + o_scan);
  const unsigned char* d_masks = d + o_mask;
  unsigned char* wk = f->d_work.as<unsigned char>();
  int* d_cnt = reinterpret_cast<int*>(wk);
  int* d_tot = reinterpret_cast<int*>(wk + o_tot);
  int* d_area = reinterpret_cast<int*>(wk + o_area);
  unsigned char* o = f->d_out.as<unsigned char>();
  int* d_hdr = reinterpret_cast<int*>(o + L.hdr);
  float* d_pts = reinterpret_cast<float*>(o + L.pts);
  float* d_rays = reinterpret_cast<float*>(o + L.rays);
  cudaStream_t st = f->stream;
  CU(cudaMemcpyAsync(d, h, in_bytes, cudaMemcpyHostToDevice, st));
  const int sel_blocks = std::max((n_chunks + kFrameWarps - 1) / kFrameWarps, 1);
  k_frame_select<0><<<sel_blocks, kFrameWarps * 32, 0, st>>>(P, d_boxes, d_scan, d_cnt, d_tot, d_pts);
  k_frame_scan_area<<<n_boxes + n_masks, 1024, 0, st>>>(P, d_cnt, d_tot, d_hdr, d_masks, d_area);
  k_frame_select<1><<<sel_blocks, kFrameWarps * 32, 0, st>>>(P, d_boxes, d_scan, d_cnt, d_tot, d_pts);
  k_frame_box<<<n_boxes, kFrameBoxThreads, 0, st>>>(P, d_boxes, d_pts, d_masks, d_bb, d_area, d_hdr, d_rays);
  CU(cudaGetLastError());
  CU(cudaMemcpyAsync(f->h_out.p, o, L.bytes, cudaMemcpyDeviceToHost, st));
  CU(cudaStreamSynchronize(st));
  const int* hh = f->h_out.as<int>();
  for (int b = 0; b < n_boxes; ++b) {
    DspgnLidarBoxOut r;
    r.n_pts = hh[b * kFrameHdr + 0];
    r.n_rays = hh[b * kFrameHdr + 1];
    r.mask = hh[b * kFrameHdr + 2];
    r.n_selected = hh[b * kFrameHdr + 3];
    f->last[b] = r;
    out[b] = r;
  }
  return 0;
}

int dspgn_lidar_frame_results(DspgnLidarFrame* f, float* points, float* depth, float* rays) {
  if (!f) return fail(DSPGN_E_ARG, "null frame");
  const int num_max = f->spec.num_lidar_max;
  const FrameOutLayout L(f->n_boxes, num_max);
  const unsigned char* h = f->h_out.as<unsigned char>();
  size_t np_ = 0, nr = 0;
  for (int b = 0; b < f->n_boxes; ++b) {
    const DspgnLidarBoxOut& r = f->last[b];
    const float* p = reinterpret_cast<const float*>(h + L.pts) + (size_t)b * num_max * 3;
    if (points) memcpy(points + 3 * np_, p, 12 * (size_t)r.n_pts);
    if (depth)
      for (int i = 0; i < r.n_pts; ++i) depth[np_ + i] = p[3 * i + 2];
    np_ += r.n_pts;
    if (r.n_rays > 0) {
      const float* q = reinterpret_cast<const float*>(h + L.rays) + (size_t)b * (num_max + kFrameBackground) * 3;
      if (rays) memcpy(rays + 3 * nr, q, 12 * (size_t)r.n_rays);
      nr += r.n_rays;
    }
  }
  return 0;
}

}  // extern "C"

// ---- A monocular keyframe's detection (dspgn_mono.cuh) ----

struct DspgnMonoFrame : FrameCore {
  DspgnMonoSpec spec{};
  int n_kp_blocks = 0;         // of the last run
  DspgnMonoOut last{-1, 0, -1, 0};
};

namespace {

// the output block of a run: header, rays [200][3], per keypoint block: count, then its passing indices
struct MonoOutLayout {
  size_t rays, cnt, idx, bytes;
  explicit MonoOutLayout(int n_kp_blocks) {
    rays = align16(4 * (size_t)kMonoHdr);
    cnt = rays + align16(12 * (size_t)kFrameBackground);
    idx = cnt + align16(4 * (size_t)n_kp_blocks);
    bytes = idx + 4 * (size_t)n_kp_blocks * kMonoKpPerBlock;
  }
};

}  // namespace

extern "C" {

int dspgn_mono_frame_create(const DspgnMonoSpec* spec, int device, DspgnMonoFrame** out) {
  if (!spec || !out) return fail(DSPGN_E_ARG, "null argument");
  if (spec->img_h < 1 || spec->img_h > 4096 || spec->img_w < 1 || spec->img_w > 4096) return fail(DSPGN_E_ARG, "image size must be in [1,4096]^2");
  if (spec->downsample_ratio < 1) return fail(DSPGN_E_ARG, "downsample_ratio must be >= 1");
  if (spec->mask_erosion < 0 || spec->mask_erosion > kMonoMaxErosion) return fail(DSPGN_E_ARG, "mask_erosion must be in [0,63]");
  if (!(spec->k[0] != 0.0 && spec->k[4] != 0.0)) return fail(DSPGN_E_ARG, "fx and fy must be nonzero");
  return frame_create(*spec, device, out);
}

void dspgn_mono_frame_destroy(DspgnMonoFrame* f) { frame_destroy(f); }

int dspgn_mono_frame_set_stream(DspgnMonoFrame* f, void* cuda_stream) { return frame_set_stream(f, cuda_stream); }

int dspgn_mono_frame_run(DspgnMonoFrame* f, const uint8_t* masks, const int32_t* bboxes, int n_masks,
                         const float* keypoints, int n_kp, DspgnMonoOut* out) {
  if (!f) return fail(DSPGN_E_ARG, "null frame");
  const DspgnMonoSpec& sp = f->spec;
  if (n_masks < 0 || n_masks > kFrameMaxMasks) return fail(DSPGN_E_ARG, "n_masks must be in [0, 64]");
  if (n_kp < 0 || n_kp > (1 << 20)) return fail(DSPGN_E_ARG, "n_kp must be in [0, 2^20]");
  if (!out || (n_masks > 0 && (!masks || !bboxes)) || (n_kp > 0 && !keypoints))
    return fail(DSPGN_E_ARG, "null pointer where data is required");
  if (int rc = check_bboxes(bboxes, n_masks, sp.img_w, sp.img_h)) return rc;
  for (int i = 0; i < n_kp; ++i) {       // cv::Mat::at reads ((int)y, (int)x): both truncations inside the image
    const float x = keypoints[2 * i], y = keypoints[2 * i + 1];
    if (!(x > -1.f && x < (float)sp.img_w && y > -1.f && y < (float)sp.img_h))
      return fail(DSPGN_E_ARG, "keypoint " + std::to_string(i) + " does not truncate to a pixel inside the image");
  }
  CU(cudaSetDevice(f->device));
  f->last = DspgnMonoOut{-1, 0, -1, 0};
  f->n_kp_blocks = 0;
  *out = f->last;
  if (n_masks == 0) return 0;              // the reference returns no instance; nothing reads the keypoints
  const int n_kp_blocks = (n_kp + kMonoKpPerBlock - 1) / kMonoKpPerBlock;
  // staged input block: bboxes | keypoints | masks (each mask padded to 16 bytes)
  const size_t mstride = align16((size_t)sp.img_h * sp.img_w);
  const size_t o_kp = align16(16 * (size_t)n_masks);
  const size_t o_mask = o_kp + align16(8 * (size_t)n_kp);
  const size_t in_bytes = o_mask + mstride * n_masks;
  const MonoOutLayout L(n_kp_blocks);
  if (f->h_in.reserve(in_bytes) || f->h_out.reserve(L.bytes)) return fail(DSPGN_E_ALLOC, "cudaMallocHost");
  if (f->d_in.reserve(in_bytes) || f->d_work.reserve(4 * kFrameMaxMasks) || f->d_out.reserve(L.bytes))
    return fail(DSPGN_E_ALLOC, "cudaMalloc");
  unsigned char* h = f->h_in.as<unsigned char>();
  memcpy(h, bboxes, 16 * (size_t)n_masks);
  if (n_kp) memcpy(h + o_kp, keypoints, 8 * (size_t)n_kp);
  stage_masks(h + o_mask, masks, n_masks, (size_t)sp.img_h * sp.img_w, mstride);
  FrameParams A{};                         // the LiDAR call's area blocks: n_boxes = 0, one block per mask
  A.n_masks = n_masks;
  A.mask_stride = (long long)mstride;
  MonoParams P{};
  memcpy(P.P, sp.k, sizeof(P.P));
  memcpy(P.inv_k, sp.inv_k, sizeof(P.inv_k));
  P.fx = sp.k[0]; P.fy = sp.k[4]; P.cx = sp.k[2]; P.cy = sp.k[5];
  P.ifx = 1. / P.fx; P.ify = 1. / P.fy;
  P.k1 = sp.k1; P.k2 = sp.k2;
  P.img_h = sp.img_h; P.img_w = sp.img_w; P.alpha = sp.downsample_ratio; P.erosion = sp.mask_erosion;
  P.n_masks = n_masks; P.n_kp = n_kp; P.mask_stride = (long long)mstride;
  unsigned char* d = f->d_in.as<unsigned char>();
  const int* d_bb = reinterpret_cast<const int*>(d);
  const float2* d_kp = reinterpret_cast<const float2*>(d + o_kp);
  const unsigned char* d_masks = d + o_mask;
  int* d_area = f->d_work.as<int>();
  unsigned char* o = f->d_out.as<unsigned char>();
  cudaStream_t st = f->stream;
  CU(cudaMemcpyAsync(d, h, in_bytes, cudaMemcpyHostToDevice, st));
  k_frame_scan_area<<<n_masks, 1024, 0, st>>>(A, nullptr, nullptr, nullptr, d_masks, d_area);
  k_mono_frame<<<1 + n_kp_blocks, kFrameBoxThreads, 0, st>>>(P, d_masks, d_bb, d_kp, d_area, reinterpret_cast<int*>(o),
                                                             reinterpret_cast<float*>(o + L.rays),
                                                             reinterpret_cast<int*>(o + L.cnt),
                                                             reinterpret_cast<int*>(o + L.idx));
  CU(cudaGetLastError());
  CU(cudaMemcpyAsync(f->h_out.p, o, L.bytes, cudaMemcpyDeviceToHost, st));
  CU(cudaStreamSynchronize(st));
  const int* hh = f->h_out.as<int>();
  const int* cnt = reinterpret_cast<const int*>(f->h_out.as<unsigned char>() + L.cnt);
  DspgnMonoOut r{hh[0], hh[1], hh[2], 0};
  for (int b = 0; b < n_kp_blocks; ++b) r.n_feature += cnt[b];
  f->n_kp_blocks = n_kp_blocks;
  f->last = r;
  *out = r;
  return 0;
}

int dspgn_mono_frame_results(DspgnMonoFrame* f, float* background_rays, int32_t* feature_idx) {
  if (!f) return fail(DSPGN_E_ARG, "null frame");
  const MonoOutLayout L(f->n_kp_blocks);
  const unsigned char* h = f->h_out.as<unsigned char>();
  if (background_rays && f->last.n_rays > 0) memcpy(background_rays, h + L.rays, 12 * (size_t)f->last.n_rays);
  if (feature_idx) {
    const int* cnt = reinterpret_cast<const int*>(h + L.cnt);
    const int* idx = reinterpret_cast<const int*>(h + L.idx);
    size_t n = 0;
    for (int b = 0; b < f->n_kp_blocks; ++b) {
      memcpy(feature_idx + n, idx + (size_t)b * kMonoKpPerBlock, 4 * (size_t)cnt[b]);
      n += cnt[b];
    }
  }
  return 0;
}

}  // extern "C"
