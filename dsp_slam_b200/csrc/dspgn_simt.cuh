// fp32 SIMT decoder engine: fused  transform -> DeepSDF forward -> backward-to-input -> Jacobian rows
// -> per-tile partial sums of J^T J / J^T r  for one tile per CTA iteration (64 rows; 32 for layers wider than 256).
// This engine is the on-device ground truth (plain FFMA, fp32 accumulation in k order) against which the tensor-core
// engine is checked.
//
// Restates: loss.py:22-43 (SDF term), loss.py:143-150 (band rows of the render term),
// loss_utils.py:51-103 (decode / input Jacobian), deep_sdf_decoder.py:75-110, optimizer.py:161-167.
#pragma once
#include <stddef.h>
#include "dspgn_common.cuh"

namespace dspgn {

constexpr int kTcRows = 128;     // rows per tile of the tensor-core engine (dspgn_tc.cuh)
constexpr int kThreads = 256;
constexpr int kHid = 256;        // max layer width of the tensor-core engine and of the narrow SIMT instantiation
constexpr int kHidWide = 512;    // max layer width of the wide SIMT instantiation (the widest decoder accepted)
// Rows per tile of the SIMT instantiation for layers up to `hid` wide: 256 threads own 8 features x 8 rows each, so
// hid x rows = 256 x 64 = 512 x 32.  Shared memory of the wide tile (SimtSmem<512>): activations 64 KB, weight chunks
// 64 KB, ReLU masks 16 KB, decoder input and its gradient 17 KB, the rest 6 KB -- 168 KB of the 227 KB opt-in.  A 64-row
// tile at 512 would need 241 KB.
__host__ __device__ constexpr int simt_rows(int hid) { return hid <= kHid ? 64 : 32; }
__host__ __device__ constexpr int ilog2(int x) { return x <= 1 ? 0 : 1 + ilog2(x >> 1); }
constexpr int kKC = 16;          // reduction chunk staged in smem
constexpr int kMaxObjScan = 1024;

struct DecoderDev {
  int L, n_lin, latent_in, in0;            // in0 = L + 3
  int in_dim[DSPGN_MAX_LINEAR], out_dim[DSPGN_MAX_LINEAR];
  // weight images at the row stride H of the SIMT instantiation that runs the class (256, or 512 in a solver that holds
  // a class wider than 256); the tensor-core engine reads them at 256
  const float* Wf[DSPGN_MAX_LINEAR];       // forward, reduction-major  [in_pad16][H]:  Wf[i*H+j] = W[j][i]
  const float* Wb[DSPGN_MAX_LINEAR];       // backward, reduction-major [out_pad16][H]: Wb[i*H+j] = W[i][j]
  const float* bias[DSPGN_MAX_LINEAR];     // [max(256, width)] zero padded
  const float* w_last;                     // [max(256, width)] last layer row
  // optional variants (deep_sdf_decoder.py:41-47,58-63,87-102): SIMT engine only
  int cat_kind[DSPGN_MAX_LINEAR];          // input of layer k = [activations | 0: nothing, 1: decoder input, 2: xyz]
  const float* ln_gamma[DSPGN_MAX_LINEAR]; // LayerNorm after layer k (nullptr = none), [max(256, width)] zero padded
  const float* ln_beta[DSPGN_MAX_LINEAR];
  int use_tanh, generic;                   // generic = any variant in use
  // tensor-core engine images (dspgn_tc.cuh): pre-swizzled fp16 hi/lo weight chunks + step plan
  const unsigned char* tc_blob;
  TcPlan tc_plan;
};

// MODE_GRIDFWD (per-launch kernels only): forward-only decode of the call-wide mesh query grid (TermArgs.grid, no pose
// transform) with each object's final code, for the objects whose record's mesh word is DSPGN_MESH_DONE; the sdf of grid
// row r of object o goes to b.sdf[grid_slot[o] * grid_rows + r]
enum { MODE_SDF = 0, MODE_BAND = 1, MODE_RAYFWD = 2, MODE_PTSFWD = 3, MODE_GRIDFWD = 4 };

// the record word that carries DSPGN_MESH_* (DspgnObjectOut.mesh)
constexpr int kRecMeshWord = 86;
__device__ __forceinline__ int record_mesh(const float* results, int o) {
  return reinterpret_cast<const int*>(results + (size_t)o * DSPGN_RESULT_FLOATS)[kRecMeshWord];
}

// Cooperative stop of a run (dspgn_keyframe_stop): the solver's host-mapped stop word holds the generation of the last
// call a stop was requested for; the run stops when it holds its own call's generation.
struct StopDev {
  unsigned* word;            // host-mapped; nullptr = the run cannot stop (no stoppable call, multi-GPU exchange, debug)
  unsigned gen;              // generation of the call the run belongs to
  int dbg_obj, dbg_iter;     // dspgn_debug_stop_at: the resident slot / iteration at whose solve the device raises the stop
  const int* pair;           // [n_obj] other hypothesis of a mono pair, -1 none (nullptr: no pair in the run)
};

// The resident batch and its run, as every kernel of the run sees it (one by-value kernel parameter; the persistent
// kernel keeps a copy in shared memory for its out-of-line solve step).
struct BatchDev {
  const ObjMeta* meta;
  ObjState* state;
  const DecoderDev* decs;
  int n_obj, n_classes;
  int D;                     // depth samples per ray
  const float* pts;          // camera-frame surface points (xyz interleaved)
  const float* rays;         // camera-frame ray directions (xyz interleaved)
  const float* depth_fg;     // observed depth of the foreground rays
  const float* T_init;       // [n_obj][16] row-major object->camera input pose
  const float* code_init;    // [n_obj][64]
  // render buffers
  float* sdf;                // per ray sample (MODE_PTSFWD: per point): sdf, +inf when outside the unit sphere
  float* band_x;             // band rows: object-frame points xyz interleaved, per-sample capacity
  float* band_s;             // de_ds per band row
  float* band_r;             // residual per band row
  int* band_m;               // band rows per object
  int* V_count;              // ray samples inside the unit sphere per object
  float* results;            // [n_obj][DSPGN_RESULT_FLOATS]
  GatherDev gather;          // optional: the record also goes straight into rank 0's HBM (peer store over NVLink)
  // per-run object table
  const int* modes;          // [n_obj] DSPGN_MODE_* of each object
  const int* q0_off;         // [n_obj] first iteration-0 slot of each object in the persistent kernel's queue
  // gated keyframe runs (nullptr = none): link[o] = the joint slot of gated pose-only object o / the pose-only object of
  // joint slot o, -1 otherwise; t_map [n_obj][16] the map's prediction of each gated object
  const int* link;
  const float* t_map;
  StopDev stop;
  // the last linearisation of every slot (dspgn_pose_information): H without damping, packed upper triangle of the slot's
  // own P x P system, (7 + code_len)(8 + code_len) / 2 floats per slot; nullptr = the run keeps none
  float* lin;
};

struct TermArgs {
  int mode;
  int iter;                  // per-iteration schedule: the iteration being evaluated (objects with n_iter <= iter are done)
  uint8_t* pt_active;        // inlier mask of the pose-only objects (optimizer.py:76-78), may be null: |res| <= 0.05 per
                             // point, written while the object runs iteration cut_iter and applied after it
  int cut_iter;              // object iteration at which the cut is recorded (4), -1 = never
  float* part;               // per-tile partial sums of this term: [tile][kAccStride] (H upper | b | loss, rows)
  int* tile_base;            // [n_obj] first tile of each object in this launch (written by CTA 0)
  float huber_b;
  // persistent kernel with the render term: the band rows' partials / tile bases / Huber threshold (SDF ones above)
  float* part_r; const int* tile_base_r; float huber_b1;
  float* ln_scratch;         // SIMT engine, LayerNorm decoders: per-CTA [layer][H][rows] normalised activations
  // debug dump of Jacobian rows (external order [pose | code]) for one object
  float* dbg_J; float* dbg_res; int dbg_obj; int dbg_P;
  // MODE_GRIDFWD: query points [grid_rows][3], grid slot of each object (-1: none)
  const float* grid; const int* grid_slot; int grid_rows;
};

// Device work queue of the persistent object-pipelined kernel (dspgn_tc.cuh).
// item = kind << 29 | object << 19 | tile   (kind: the tile's MODE_*; object < 1024; tile < 2^19; always >= 0)
// A queue slot is ONE word: 0 = not published yet, item + 1 = published (payload and flag in one store / one load).
constexpr int kItemKindShift = 29, kItemObjShift = 19, kItemTileMask = (1 << 19) - 1, kItemObjMask = 1023;
constexpr int kKindScan = 3;   // queue-only kind: per-ray scan of a 64-ray chunk (no GEMM steps); 0..2 = MODE_SDF / MODE_BAND / MODE_RAYFWD
__host__ __device__ __forceinline__ int make_item(int kind, int o, int tile) {
  return (kind << kItemKindShift) | (o << kItemObjShift) | tile;
}
// filler for reserved queue slots that turned out not to be needed (k_init reserves every object's iteration-0 slots
// from host-side upper bounds): consumers skip it.  Never a real item (a scan item's tile index is < 128); + 1 fits an int.
constexpr int kItemNop = 0x7ffffffe;

// Counters of the work queue: one device block, read back whole by dspgn_results.  The contended atomics (head, tail,
// done_objects, abort_flag) sit 128 bytes apart.
struct QueueCounters {
  int head; int pad0_[31];          // consumer ticket counter
  int tail; int pad1_[31];          // producer reservation counter
  int done_objects; int pad2_[15];  // objects finished (last iteration or frozen)
  int band_rows_total; int pad3_[7];          // sum of band rows over all objects and iterations (roofline accounting)
  unsigned long long valid_rows_total; int pad4_[6];   // sum of V (ray samples inside the unit sphere), same
  int abort_flag; int pad5_[31];    // set when a queue wait timed out: every CTA drains and exits (soft failure, never a trap)
};
static_assert(offsetof(QueueCounters, head) == 4 * 0 && offsetof(QueueCounters, tail) == 4 * 32 &&
              offsetof(QueueCounters, done_objects) == 4 * 64 && offsetof(QueueCounters, band_rows_total) == 4 * 80 &&
              offsetof(QueueCounters, valid_rows_total) == 4 * 88 && offsetof(QueueCounters, abort_flag) == 4 * 96 &&
              sizeof(QueueCounters) == 4 * 128, "queue counter layout");

// Optional event log of the persistent kernel (env DSPGN_CLK): ev[0] = count, then per event {%globaltimer ns,
// descriptor kind<<56 | mode<<52 | sm<<40 | object<<24 | tile (or iteration / solve phase)}.
struct EventLog { long long* ev; int cap; };
enum { EV_TILE_BEGIN = 0, EV_TILE_END = 1, EV_SCAN_BEGIN = 2, EV_SCAN_END = 3, EV_SOLVE_BEGIN = 4, EV_SOLVE_END = 5, EV_POPPED = 6,
       EV_FIRST_MMA = 7, EV_SOLVE_PHASE = 8 };
__device__ __forceinline__ long long ev_desc(int kind, int mode, int o, int tile) {
  return ((long long)kind << 56) | ((long long)mode << 52) | ((long long)o << 24) | (long long)tile;
}
// the writer adds the SM to the descriptor
__device__ __forceinline__ void log_event(const EventLog& log, long long desc) {
  if (log.ev == nullptr) return;
  const unsigned long long slot = atomicAdd(reinterpret_cast<unsigned long long*>(log.ev), 1ull);
  if ((long long)slot >= log.cap) return;
  unsigned long long t; unsigned sm;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  asm volatile("mov.u32 %0, %%smid;" : "=r"(sm));
  log.ev[1 + 2 * slot] = (long long)t;
  log.ev[2 + 2 * slot] = desc | ((long long)sm << 40);
}

struct MegaArgs {
  int q_cap;                 // total items that can ever be pushed
  int render;                // 1: the joint objects run the render term (ray-sample tiles -> per-ray scan -> band tiles)
  int total0;                // iteration-0 slots, seeded by k_init (the initial tail)
  int* q_flag;               // one word per slot (no wrap-around): 0 = empty, item + 1 = published
  QueueCounters* ctr;
  int* pending;              // [n_obj] SDF + band tiles of the object's current iteration still running (+1 while the
                             //         render term has not been expanded into band tiles yet)
  int* ray_left;             // [n_obj] ray-sample tiles of the current iteration still running
  int* scan_left;            // [n_obj] scan items (64-ray chunks) of the current iteration still running
  int* seg_cnt; int* seg_prefix;   // band rows kept per 8-ray segment / their exclusive prefix per object (dspgn_solve.cuh)
  int* obj_iter;             // [n_obj] current iteration of each object
  int* vpre;                 // per ray: (exclusive prefix of the valid-sample hulls << kRangeSampleBits) | first valid
                             // sample, n_rays + 1
                             // entries per object at ray_off + o (dspgn_solve.cuh: valid_sample_ranges); nullptr = the
                             // forward-only tiles enumerate all n_rays * D samples
  EventLog log;
};

// ---------------------------------------------------------------------------------------------
// tile scheduling shared by all decoder kernels: rows per object -> tiles, scanned per CTA
__device__ __forceinline__ int term_rows(const BatchDev& b, const TermArgs& a, int o) {
  if (a.mode == MODE_GRIDFWD) return (record_mesh(b.results, o) == DSPGN_MESH_DONE) ? a.grid_rows : 0;
  const ObjState& st = b.state[o];
  if (st.status != 0 || a.iter >= st.n_iter) return 0;
  if (a.mode == MODE_SDF || a.mode == MODE_PTSFWD) return b.meta[o].n_pts;
  if (st.mode != DSPGN_MODE_JOINT) return 0;          // pose-only objects have no render term
  if (a.mode == MODE_BAND) return b.band_m[o];
  return b.meta[o].n_rays * b.D;
}

// SDF rows of a pose-only object: raw residuals (optimizer.py:71), otherwise the term's Huber threshold
__device__ __forceinline__ float term_huber(const TermArgs& a, int term, int obj_mode, float b) {
  return (term == MODE_SDF && obj_mode == DSPGN_MODE_POSE) ? INFINITY : b;
}

// inlier cut of a pose-only object at object iteration `it` (optimizer.py:76-78): the mask it reads / writes, or null
__device__ __forceinline__ void cut_masks(const TermArgs& a, int obj_mode, int it, const uint8_t*& in, uint8_t*& out) {
  const bool on = a.pt_active != nullptr && a.cut_iter >= 0 && obj_mode == DSPGN_MODE_POSE;
  in = (on && it > a.cut_iter) ? a.pt_active : nullptr;
  out = (on && it == a.cut_iter) ? a.pt_active : nullptr;
}

// ---- per-row stages of every tile body (simt_tile, tc_body, tcw_body) ----------------------------------------------
// Band row `row` of an object on the persistent schedule: band rows live compacted per ray segment (scan_prefix), so the
// row is in the largest segment lo whose prefix segp[lo] <= row.  Its sample index, from the object's first sample `base`;
// seg_samples = ray samples per segment (kSegRays x D).
__device__ __forceinline__ size_t band_row_sample(const int* segp, int nseg, size_t base, size_t seg_samples, int row) {
  int lo = 0, hi = nseg;
  while (hi - lo > 1) { const int mid = (lo + hi) >> 1; if (segp[mid] <= row) lo = mid; else hi = mid; }
  return base + (size_t)lo * seg_samples + (size_t)(row - segp[lo]);
}

// Ray-sample row `row` of object M: sample j of ray `ray` at depth lin_depth(dmin, dmax, dstep, j), in the object frame
// through T (T_oc); returns its weight, 1 inside the unit sphere (loss.py:68).  Rows are ray * D + j, or with `compact`
// they enumerate the valid-sample hulls: hull[ray] = first row << kRangeSampleBits | first sample, and the row belongs
// to the largest ray whose hull starts at or before it.
__device__ __forceinline__ float ray_sample_row(const BatchDev& b, const ObjMeta& M, const float* T, float dmin, float dmax,
                                                float dstep, const int* hull, bool compact, int row, float& x0, float& x1,
                                                float& x2) {
  int ray = row / b.D, j = row - ray * b.D;
  if (compact) {
    int lo = 0, hi = M.n_rays;
    while (hi - lo > 1) { const int mid = (lo + hi) >> 1; if ((hull[mid] >> kRangeSampleBits) <= row) lo = mid; else hi = mid; }
    ray = lo; j = (hull[lo] & kRangeSampleMask) + (row - (hull[lo] >> kRangeSampleBits));
  }
  const float* rq = b.rays + 3 * (size_t)(M.ray_off + ray);
  const float d = lin_depth(dmin, dmax, dstep, j, b.D);
  xform_point(T, __fmul_rn(rq[0], d), __fmul_rn(rq[1], d), __fmul_rn(rq[2], d), x0, x1, x2);
  return inside_unit_sphere(x0, x1, x2) ? 1.f : 0.f;
}

struct RowTail { float rho_r, n, res; };
// The end of tile row r's Jacobian row J (column c at J[c * cs]; columns 64..66 hold the input gradient g), thread = row:
// pose columns  dsdf/dx . [I | -x^ | x] = [g, x cross g, g.x]  at the object-frame point x (loss_utils.py:166-185; no
// scale column for a pose-only object) and column 71 zeroed; the residual of the row (res: the decoder output of an SDF
// row, the residual of a band row; 0 for a padded or masked-out row) and the inlier-cut mask of an SDF row at
// mask_out[mask_base + r] (optimizer.py:76-78).  Returns rho r (loss_utils.py:250-265, threshold huber_b), the row's
// count in the loss's row count and the raw residual.  (mask_base: the object's first point + the tile's first row;
// with the row index added here, k_decoder_tc keeps its register allocation.)
__device__ __forceinline__ RowTail row_tail(float* J, int cs, float x0, float x1, float x2, float g0, float g1, float g2,
                                            float res, float sc, int r, int nrows, int mode, int omode, float huber_b,
                                            uint8_t* mask_out, int mask_base) {
  J[(kMaxCode + 3) * cs] = x1 * g2 - x2 * g1;
  J[(kMaxCode + 4) * cs] = x2 * g0 - x0 * g2;
  J[(kMaxCode + 5) * cs] = x0 * g1 - x1 * g0;
  J[(kMaxCode + 6) * cs] = (omode == DSPGN_MODE_POSE) ? 0.f : (g0 * x0 + g1 * x1 + g2 * x2);
  J[(kMaxCode + 7) * cs] = 0.f;
  if (sc == 0.f && (mode == MODE_SDF || r >= nrows)) res = 0.f;
  if (mask_out != nullptr && mode == MODE_SDF && r < nrows)
    mask_out[mask_base + r] = (sc != 0.f && fabsf(res) <= 0.05f) ? 1 : 0;
  return {huber_weight(fabsf(res), huber_b) * res, (mode == MODE_SDF) ? sc : (r < nrows ? 1.f : 0.f), res};
}

// Debug hook: rows 0 .. nrows-1 of the tile's Jacobian (row p, column c at J[p * rs + c * cs]) into a.dbg_J at tile row
// row0, P columns each, pose columns first
__device__ __forceinline__ void dbg_dump_J(const TermArgs& a, const float* J, int rs, int cs, int row0, int nrows, int omode,
                                           int tid, int nthreads) {
  const int P = a.dbg_P, npose = (omode == DSPGN_MODE_POSE) ? 6 : 7;
  for (int idx = tid; idx < nrows * P; idx += nthreads) {
    const int p = idx / P, c = idx - p * P;
    const int ci = (c < npose) ? (kMaxCode + c) : (c - npose);
    a.dbg_J[(size_t)(row0 + p) * P + c] = J[p * rs + ci * cs];
  }
}

// exclusive scan of tiles per object into s_prefix[0..n_obj]; returns total (all threads)
__device__ inline int build_tile_prefix(const BatchDev& b, const TermArgs& a, int tile_rows, int* s_prefix, int* s_warp) {
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nw = blockDim.x >> 5;
  int carry = 0;
  for (int base = 0; base < b.n_obj; base += blockDim.x) {
    int o = base + tid;
    int v = (o < b.n_obj) ? (term_rows(b, a, o) + tile_rows - 1) / tile_rows : 0;
    int x = v;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) { int y = __shfl_up_sync(0xffffffffu, x, d); if (lane >= d) x += y; }
    if (lane == 31) s_warp[warp] = x;
    __syncthreads();
    int woff = 0;
    for (int w = 0; w < warp; ++w) woff += s_warp[w];
    int tot = 0;
    for (int w = 0; w < nw; ++w) tot += s_warp[w];
    if (o < b.n_obj) s_prefix[o] = carry + woff + x - v;
    carry += tot;
    __syncthreads();
  }
  if (tid == 0) s_prefix[b.n_obj] = carry;
  __syncthreads();
  if (blockIdx.x == 0 && a.tile_base != nullptr)
    for (int o = tid; o < b.n_obj; o += blockDim.x) a.tile_base[o] = s_prefix[o];
  return carry;
}

__device__ __forceinline__ int find_object(const int* s_prefix, int n_obj, int tile) {
  int lo = 0, hi = n_obj;      // largest o with prefix[o] <= tile
  while (hi - lo > 1) { int mid = (lo + hi) >> 1; if (s_prefix[mid] <= tile) lo = mid; else hi = mid; }
  return lo;
}

// A tile of kind `mode` runs the decoder forward only (ray-sample, point-forward and grid-forward tiles).  MEGA: the
// persistent schedule, whose queue kind 3 is a scan item (kKindScan), not MODE_PTSFWD.
template <bool MEGA>
__device__ __forceinline__ bool tile_fwd_only(int mode) {
  return mode == MODE_RAYFWD || (!MEGA && (mode == MODE_PTSFWD || mode == MODE_GRIDFWD));
}
// GEMM steps of a tensor-core tile of kind `mode` with step plan p: none for a scan item, the forward steps for a
// forward-only tile, every step otherwise
template <bool MEGA>
__device__ __forceinline__ int tile_steps(const TcPlan& p, int mode) {
  if (MEGA && mode == kKindScan) return 0;
  return tile_fwd_only<MEGA>(mode) ? p.n_fwd : p.n_steps;
}

// The object of the tile being run, staged in shared memory by its prologue (stage_obj, dspgn_tc.cuh)
struct TileObj {
  float ost[16];                     // T_oc[12], dmin, dmax, dstep, dfar
  float zs[kMaxCode + 16];           // latent code, zero padded
};

// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ void cp_async16(void* smem, const void* gmem) {
  uint32_t s = (uint32_t)__cvta_generic_to_shared(smem);
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(s), "l"(gmem) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N> __device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

// acc[jj][pp] = sum_{i<Kred} Wg[i*H + 8*jg+jj] * in_s[i*TP + 8*pg+pp]
template <int H, int TP>
__device__ __forceinline__ void gemm_rm(const float* __restrict__ Wg, int Kred, const float* __restrict__ in_s,
                                        float* __restrict__ wbuf, float (&acc)[8][8]) {
  constexpr int kLoads = kKC * H / 4 / kThreads;     // 16-byte copies per thread and weight chunk
  const int tid = threadIdx.x, jg = tid >> ilog2(TP / 8), pg = tid & (TP / 8 - 1);
#pragma unroll
  for (int a = 0; a < 8; ++a)
#pragma unroll
    for (int b = 0; b < 8; ++b) acc[a][b] = 0.f;
  const int nch = (Kred + kKC - 1) / kKC;
  // prefetch chunk 0
  {
    const float4* src = reinterpret_cast<const float4*>(Wg);
    float4* dst = reinterpret_cast<float4*>(wbuf);
#pragma unroll
    for (int q = 0; q < kLoads; ++q) cp_async16(dst + tid + q * kThreads, src + tid + q * kThreads);
    cp_async_commit();
  }
  for (int c = 0; c < nch; ++c) {
    cp_async_wait<0>();
    __syncthreads();                 // chunk c landed for all; everyone is done with chunk c-1's buffer
    if (c + 1 < nch) {
      const float4* src = reinterpret_cast<const float4*>(Wg + (size_t)(c + 1) * kKC * H);
      float4* dst = reinterpret_cast<float4*>(wbuf + ((c + 1) & 1) * kKC * H);
#pragma unroll
      for (int q = 0; q < kLoads; ++q) cp_async16(dst + tid + q * kThreads, src + tid + q * kThreads);
      cp_async_commit();
    }
    const float* wb = wbuf + (c & 1) * kKC * H + 8 * jg;
    const float* ib = in_s + (size_t)c * kKC * TP + 8 * pg;
    const int kmax = min(kKC, Kred - c * kKC);
#pragma unroll 4
    for (int kk = 0; kk < kmax; ++kk) {
      float4 w0 = *reinterpret_cast<const float4*>(wb + kk * H);
      float4 w1 = *reinterpret_cast<const float4*>(wb + kk * H + 4);
      float4 a0 = *reinterpret_cast<const float4*>(ib + kk * TP);
      float4 a1 = *reinterpret_cast<const float4*>(ib + kk * TP + 4);
      const float w[8] = {w0.x, w0.y, w0.z, w0.w, w1.x, w1.y, w1.z, w1.w};
      const float x[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
#pragma unroll
      for (int a = 0; a < 8; ++a)
#pragma unroll
        for (int b = 0; b < 8; ++b) acc[a][b] = fmaf(w[a], x[b], acc[a][b]);
    }
  }
  __syncthreads();                   // all reads of in_s / wbuf finished: caller may overwrite in_s
}

template <int H>
struct SimtSmem {
  static constexpr int TP = simt_rows(H);
  float act[H * TP];                 // feature-major activations / gradients / J rows
  float inp[(kMaxCode + 4) * TP];    // decoder input [z | x] rows
  float gin[(kMaxCode + 4) * TP];    // d sdf / d(input) collected from the concat layers (latent_in / xyz_in_all)
  float lnst[DSPGN_MAX_LINEAR * TP];        // LayerNorm: [layer][p] reciprocal std (the mean is not needed backward)
  float wbuf[2 * kKC * H];
  uint8_t mask[8 * H * (TP / 8)];    // ReLU masks: [layer][feature][p/8] bit p%8
  float xo[3 * TP];
  float yv[TP], rr[TP], rscale[TP];
  float red[kThreads];               // last layer: one partial dot product per thread
  TileObj obj;
  int prefix[kMaxObjScan + 1];
  int warp_tmp[32];
};
static_assert(sizeof(SimtSmem<kHidWide>) <= 227 * 1024, "wide SIMT tile exceeds the opt-in shared memory");

// LayerNorm backward (deep_sdf_decoder.py:96-102 through autograd): S.act holds the gradient w.r.t. the LN OUTPUT of
// `layer` for its n features (already through the ReLU mask); turn it into the gradient w.r.t. the LN input:
//   g_x = rstd * (gamma g - mean_j(gamma g) - xhat * mean_j(gamma g xhat)).     All threads; caller has synchronised.
template <int TP>
__device__ inline void simt_ln_backward(float* act, float* red, const float* rstd, const float* __restrict__ gamma,
                                        const float* __restrict__ xhat, int n) {
  const int tid = threadIdx.x;
  if (tid < TP) {
    float s1 = 0.f, s2 = 0.f;
    for (int j = 0; j < n; ++j) {
      const float gg = act[j * TP + tid] * gamma[j];
      s1 += gg;
      s2 = fmaf(gg, xhat[j * TP + tid], s2);
    }
    red[tid] = s1 / (float)n;
    red[TP + tid] = s2 / (float)n;
  }
  __syncthreads();
  for (int idx = tid; idx < n * TP; idx += kThreads) {
    const int j = idx / TP, p = idx - j * TP;
    const float gg = act[idx] * gamma[j];
    act[idx] = rstd[p] * (gg - red[p] - xhat[idx] * red[TP + p]);
  }
  __syncthreads();
}

// What the persistent kernel (dspgn_simt_persistent.cuh) hands a tile beyond its object, first row, partial-sum slot and
// kind: the values other CTAs write during the run, read cache-bypassing by the kernel and staged in shared memory.
struct SimtMegaTile {
  int term_rows;             // rows of the tile's term: SDF points, ray samples (valid-sample hulls) or band rows
  int iter;                  // the object's current iteration (inlier cut)
  const int* segp;           // range words of a ray-sample tile (vpre) or a band tile (segment prefix)
  int nseg;                  // band tile: ray segments of the object
  int seg_samples;           // band tile: ray samples per segment (kSegRays x D)
  bool compact;              // ray-sample tile rows enumerate the valid-sample hulls (vpre words in segp)
};

// One tile of the SIMT engine: transform, forward, backward to the input, Jacobian rows and the tile's partial sums into
// slot `tile` of its term.  Both schedules run it: MEGA = false is k_decoder_simt (one launch per term and iteration,
// the term is a.mode), MEGA = true is k_simt_persistent (every item kind of the device queue, the kind is `mode_mega`;
// `mt` carries the values other CTAs write during the run).  The caller has staged the object in S.obj (stage_obj).  A
// row's values do not depend on which other rows share its tile.
template <int H, bool MEGA>
__device__ __forceinline__ void simt_tile(SimtSmem<H>& S, const BatchDev& b, const TermArgs& a, const int o, const int row0,
                                          const int tile, const int mode_mega, const SimtMegaTile& mt) {
  constexpr int kTP = simt_rows(H);
  constexpr int kNPart = kThreads / kTP;      // last layer: partial dot products per row
  const int tid = threadIdx.x, jg = tid >> ilog2(kTP / 8), pg = tid & (kTP / 8 - 1);
  // the tile's kind: the launch's term (read from the argument where it is used, as before the split), or the item's
  auto tmode = [&] { if constexpr (MEGA) return mode_mega; else return a.mode; };
  {
    const ObjMeta M = b.meta[o];
    const ObjState& st = b.state[o];
    const DecoderDev& dec = b.decs[M.class_id];
    const int L = dec.L, in0 = dec.in0, nl = dec.n_lin;
    const int nrows = min(kTP, (MEGA ? mt.term_rows : term_rows(b, a, o)) - row0);
    const int omode = st.mode;
    const uint8_t* mask_in; uint8_t* mask_out;
    cut_masks(a, omode, MEGA ? mt.iter : a.iter, mask_in, mask_out);

    // ---- phase 0: points in the object frame, decoder input rows -----------------------------
    if (tid < kTP) {
      const int p = tid, r = row0 + p;
      float x = 0.f, y = 0.f, z = 0.f, sc = 0.f, res = 0.f;
      if (p < nrows) {
        if (tmode() == MODE_SDF || (!MEGA && tmode() == MODE_PTSFWD)) {
          const float* q = b.pts + 3 * (size_t)(M.pts_off + r);
          xform_point(S.obj.ost, q[0], q[1], q[2], x, y, z);
          sc = (mask_in == nullptr || (MEGA ? __ldcg(mask_in + M.pts_off + r) : mask_in[M.pts_off + r])) ? 1.f : 0.f;
        } else if (!MEGA && tmode() == MODE_GRIDFWD) {
          const float* q = a.grid + 3 * (size_t)r;
          x = q[0]; y = q[1]; z = q[2]; sc = 1.f;
        } else if (tmode() == MODE_BAND) {
          if constexpr (MEGA) {
            const size_t s = band_row_sample(mt.segp, mt.nseg, M.smp_off, mt.seg_samples, r);
            x = __ldcg(b.band_x + 3 * s); y = __ldcg(b.band_x + 3 * s + 1); z = __ldcg(b.band_x + 3 * s + 2);
            sc = __ldcg(b.band_s + s); res = __ldcg(b.band_r + s);
          } else {
            const size_t s = (size_t)M.smp_off + r;
            x = b.band_x[3 * s]; y = b.band_x[3 * s + 1]; z = b.band_x[3 * s + 2];
            sc = b.band_s[s]; res = b.band_r[s];
          }
        } else {
          sc = ray_sample_row(b, M, S.obj.ost, S.obj.ost[12], S.obj.ost[13], S.obj.ost[14], mt.segp, MEGA && mt.compact, r, x,
                              y, z);
        }
      }
      S.xo[p] = x; S.xo[kTP + p] = y; S.xo[2 * kTP + p] = z;
      S.rscale[p] = sc; S.rr[p] = res;
    }
    for (int idx = tid; idx < L * kTP; idx += kThreads) S.inp[idx] = S.obj.zs[idx / kTP];
    for (int idx = tid; idx < (kMaxCode + 4) * kTP; idx += kThreads) S.gin[idx] = 0.f;
    float* const xhat_all = (a.ln_scratch != nullptr) ? a.ln_scratch + (size_t)blockIdx.x * DSPGN_MAX_LINEAR * H * kTP : nullptr;
    __syncthreads();
    if (tid < 3 * kTP) S.inp[L * kTP + tid] = S.xo[tid];
    if (tmode() == MODE_RAYFWD) {
      // whole tile outside the unit sphere: nothing to decode
      int any = __syncthreads_or(tid < kTP && S.rscale[tid] != 0.f);
      if (!any) {
        if (tid < nrows) b.sdf[(size_t)M.smp_off + row0 + tid] = INFINITY;
        __syncthreads();
        return;
      }
    } else {
      __syncthreads();
    }

    float acc[8][8];
    // ---- phase 1: forward -------------------------------------------------------------------
    for (int k = 0; k < nl - 1; ++k) {
      gemm_rm<H, kTP>(dec.Wf[k], dec.in_dim[k], (k == 0) ? S.inp : S.act, S.wbuf, acc);
      const int nout = dec.out_dim[k];
      const float* bias = dec.bias[k];
      const float* lng = dec.ln_gamma[k];
      if (lng == nullptr) {
#pragma unroll
        for (int jj = 0; jj < 8; ++jj) {
          const int j = 8 * jg + jj;
          if (j < nout) {
            const float bj = bias[j];
            unsigned bits = 0;
            float v[8];
#pragma unroll
            for (int pp = 0; pp < 8; ++pp) {
              float t = acc[jj][pp] + bj;
              bits |= (t > 0.f ? 1u : 0u) << pp;
              v[pp] = fmaxf(t, 0.f);
            }
            S.mask[(k * H + j) * (kTP / 8) + pg] = (uint8_t)bits;
            float4* dst = reinterpret_cast<float4*>(S.act + j * kTP + 8 * pg);
            dst[0] = make_float4(v[0], v[1], v[2], v[3]);
            dst[1] = make_float4(v[4], v[5], v[6], v[7]);
          }
        }
      } else {
        // ---- LayerNorm between the layer and its ReLU (deep_sdf_decoder.py:96-103), eps = 1e-5, biased variance ----
        const float* lnb = dec.ln_beta[k];
#pragma unroll
        for (int jj = 0; jj < 8; ++jj) {
          const int j = 8 * jg + jj;
          if (j < nout) {
            const float bj = bias[j];
            float4* dst = reinterpret_cast<float4*>(S.act + j * kTP + 8 * pg);
            dst[0] = make_float4(acc[jj][0] + bj, acc[jj][1] + bj, acc[jj][2] + bj, acc[jj][3] + bj);
            dst[1] = make_float4(acc[jj][4] + bj, acc[jj][5] + bj, acc[jj][6] + bj, acc[jj][7] + bj);
          }
        }
        __syncthreads();
        if (tid < kTP) {
          float m = 0.f;
          for (int j = 0; j < nout; ++j) m += S.act[j * kTP + tid];
          m /= (float)nout;
          float var = 0.f;
          for (int j = 0; j < nout; ++j) { const float d = S.act[j * kTP + tid] - m; var = fmaf(d, d, var); }
          var /= (float)nout;
          S.red[tid] = m;
          S.lnst[k * kTP + tid] = 1.0f / sqrtf(var + 1e-5f);
        }
        __syncthreads();
        float* xh_out = xhat_all + (size_t)k * H * kTP;
#pragma unroll
        for (int jj = 0; jj < 8; ++jj) {
          const int j = 8 * jg + jj;
          if (j < nout) {
            const float gj = lng[j], bj = lnb[j];
            unsigned bits = 0;
            float v[8], xh[8];
#pragma unroll
            for (int pp = 0; pp < 8; ++pp) {
              const int p = 8 * pg + pp;
              xh[pp] = (S.act[j * kTP + p] - S.red[p]) * S.lnst[k * kTP + p];
              const float t = fmaf(xh[pp], gj, bj);
              bits |= (t > 0.f ? 1u : 0u) << pp;
              v[pp] = fmaxf(t, 0.f);
            }
            S.mask[(k * H + j) * (kTP / 8) + pg] = (uint8_t)bits;
            float4* dst = reinterpret_cast<float4*>(S.act + j * kTP + 8 * pg);
            dst[0] = make_float4(v[0], v[1], v[2], v[3]);
            dst[1] = make_float4(v[4], v[5], v[6], v[7]);
            float4* xd = reinterpret_cast<float4*>(xh_out + j * kTP + 8 * pg);      // for the backward pass (L2-resident scratch)
            xd[0] = make_float4(xh[0], xh[1], xh[2], xh[3]);
            xd[1] = make_float4(xh[4], xh[5], xh[6], xh[7]);
          }
        }
      }
      if (dec.cat_kind[k + 1] == 1)          // deep_sdf_decoder.py:87-88: x = cat[x, input]
        for (int idx = tid; idx < in0 * kTP; idx += kThreads) S.act[nout * kTP + idx] = S.inp[idx];
      else if (dec.cat_kind[k + 1] == 2)     // deep_sdf_decoder.py:89-90: x = cat[x, xyz]
        for (int idx = tid; idx < 3 * kTP; idx += kThreads) S.act[nout * kTP + idx] = S.inp[L * kTP + idx];
      __syncthreads();
    }
    {  // last layer (out = 1) + tanh
      const int kin = dec.in_dim[nl - 1];
      const int p = tid & (kTP - 1), part = tid >> ilog2(kTP);
      const int j0 = part * (H / kNPart), j1 = min(kin, j0 + H / kNPart);
      float s = 0.f;
      for (int j = j0; j < j1; ++j) s = fmaf(dec.w_last[j], S.act[j * kTP + p], s);
      S.red[part * kTP + p] = s;
      __syncthreads();
      if (tid < kTP) {
        float t = S.red[tid];
#pragma unroll
        for (int q = 1; q < kNPart; ++q) t += S.red[q * kTP + tid];
        t += dec.bias[nl - 1][0];
        float dfac = 1.f;
        if (dec.use_tanh) { t = tanhf(t); dfac = 1.f - t * t; }        // deep_sdf_decoder.py:93-94
        const float y = tanhf(t);                                       // :107-108
        S.yv[tid] = y;
        S.red[tid] = (1.f - y * y) * dfac;                              // d sdf / d(last layer output)
      }
      __syncthreads();
    }
    if (tile_fwd_only<MEGA>(tmode())) {
      int cnt = 0;
      if (tid < nrows) {
        const bool valid = S.rscale[tid] != 0.f;
        const size_t base = (tmode() == MODE_RAYFWD) ? (size_t)M.smp_off
                            : (tmode() == MODE_GRIDFWD ? (size_t)a.grid_slot[o] * a.grid_rows : (size_t)M.pts_off);
        b.sdf[base + row0 + tid] = valid ? S.yv[tid] : INFINITY;
        cnt = valid ? 1 : 0;
      }
      if constexpr (!MEGA) {       // (persistent kernel: V is counted by the scan items, scan_chunk)
        cnt = __syncthreads_count(cnt);
        if (tid == 0 && cnt && tmode() == MODE_RAYFWD) atomicAdd(b.V_count + o, cnt);
      }
      return;
    }

    // ---- phase 2: backward to the input ------------------------------------------------------
    {  // seed: g = (1 - y^2) W_last, masked by the last hidden ReLU
      const int kin = dec.in_dim[nl - 1];
      const int ckl = dec.cat_kind[nl - 1];                                // the last layer's input may carry a concat too
      const int ncl = kin - (ckl == 1 ? in0 : (ckl == 2 ? 3 : 0));
      for (int idx = tid; idx < kin * kTP; idx += kThreads) {
        const int j = idx / kTP, p = idx - j * kTP;
        const float g = S.red[p] * dec.w_last[j];
        if (j < ncl) {
          const unsigned bit = (S.mask[((nl - 2) * H + j) * (kTP / 8) + (p >> 3)] >> (p & 7)) & 1u;
          S.act[idx] = bit ? g : 0.f;
        } else {
          S.gin[((ckl == 1 ? 0 : L) + (j - ncl)) * kTP + p] += g;
        }
      }
      __syncthreads();
      if (dec.ln_gamma[nl - 2] != nullptr)
        simt_ln_backward<kTP>(S.act, S.red + kTP, S.lnst + (nl - 2) * kTP, dec.ln_gamma[nl - 2], xhat_all + (size_t)(nl - 2) * H * kTP, ncl);
    }
    for (int k = nl - 2; k >= 0; --k) {
      gemm_rm<H, kTP>(dec.Wb[k], dec.out_dim[k], S.act, S.wbuf, acc);
      const int nin = dec.in_dim[k];
      const int ck = dec.cat_kind[k];
      const int ncont = (ck == 1) ? nin - in0 : (ck == 2 ? nin - 3 : nin);   // columns that continue down the chain
#pragma unroll
      for (int jj = 0; jj < 8; ++jj) {
        const int j = 8 * jg + jj;
        if (j >= nin) continue;
        float v[8];
#pragma unroll
        for (int pp = 0; pp < 8; ++pp) v[pp] = acc[jj][pp];
        float* dst;
        if (j >= ncont) {                       // concat path (latent_in: whole input, xyz_in_all: xyz) -> d/d(input)
          dst = S.gin + ((ck == 1 ? 0 : L) + (j - ncont)) * kTP + 8 * pg;
#pragma unroll
          for (int pp = 0; pp < 8; ++pp) v[pp] += dst[pp];
        } else if (k > 0) {
          const unsigned bits = S.mask[((k - 1) * H + j) * (kTP / 8) + pg];
#pragma unroll
          for (int pp = 0; pp < 8; ++pp) v[pp] = ((bits >> pp) & 1u) ? v[pp] : 0.f;
          dst = S.act + j * kTP + 8 * pg;
        } else {                                // k == 0: d/d(input) complete; scale rows (loss.py:145)
          const int jrow = (j < L) ? j : (kMaxCode + (j - L));
          dst = S.act + jrow * kTP + 8 * pg;
#pragma unroll
          for (int pp = 0; pp < 8; ++pp) {
            const float t = v[pp] + S.gin[j * kTP + 8 * pg + pp];
            v[pp] = t * S.rscale[8 * pg + pp];
          }
        }
        reinterpret_cast<float4*>(dst)[0] = make_float4(v[0], v[1], v[2], v[3]);
        reinterpret_cast<float4*>(dst)[1] = make_float4(v[4], v[5], v[6], v[7]);
      }
      __syncthreads();
      if (k > 0 && dec.ln_gamma[k - 1] != nullptr)      // through the LayerNorm of layer k-1 (its ReLU mask is applied above)
        simt_ln_backward<kTP>(S.act, S.red, S.lnst + (k - 1) * kTP, dec.ln_gamma[k - 1], xhat_all + (size_t)(k - 1) * H * kTP, ncont);
    }
    // ---- phase 3: Jacobian rows  J = [code (0..63) | pose (64..70) | 0] ---------------------------
    for (int idx = tid + L * kTP; idx < kMaxCode * kTP; idx += kThreads) S.act[idx] = 0.f;  // code_len < 64
    if (tid < kTP) {
      const int p = tid;
      const RowTail t = row_tail(S.act + p, kTP, S.xo[p], S.xo[kTP + p], S.xo[2 * kTP + p], S.act[(kMaxCode + 0) * kTP + p],
                                 S.act[(kMaxCode + 1) * kTP + p], S.act[(kMaxCode + 2) * kTP + p],
                                 (tmode() == MODE_SDF) ? S.yv[p] : S.rr[p], S.rscale[p], p, nrows, tmode(), omode,
                                 term_huber(a, tmode(), omode, (MEGA && tmode() == MODE_BAND) ? a.huber_b1 : a.huber_b),
                                 mask_out, M.pts_off + row0);
      S.yv[p] = t.res;                                      // raw residual (debug dump)
      S.rr[p] = t.rho_r;
    }
    __syncthreads();
    if (!MEGA && a.dbg_J != nullptr && o == a.dbg_obj && tmode() == MODE_SDF) {
      dbg_dump_J(a, S.act, 1, kTP, row0, nrows, omode, tid, kThreads);
      if (tid < nrows) a.dbg_res[row0 + tid] = S.yv[tid];
    }
    // ---- phase 4: H += J^T J, b += J^T (rho r), loss += sum (rho r)^2  (optimizer.py:161-167) ----
    float* accp = ((MEGA && tmode() == MODE_BAND) ? a.part_r : a.part) + (size_t)tile * kAccStride;
    if (tid < 171) {
      // upper-triangular 4x4 blocks of the 72x72 matrix: tid -> (bi <= bj)
      int bi = 0, rem = tid;
      while (rem >= 18 - bi) { rem -= 18 - bi; ++bi; }
      const int bj = bi + rem;
      float h[4][4];
#pragma unroll
      for (int u = 0; u < 4; ++u)
#pragma unroll
        for (int v = 0; v < 4; ++v) h[u][v] = 0.f;
      const float* ra = S.act + (4 * bi) * kTP;
      const float* rb = S.act + (4 * bj) * kTP;
      for (int p = 0; p < kTP; p += 4) {
        float4 A4[4], B4[4];
#pragma unroll
        for (int u = 0; u < 4; ++u) {
          A4[u] = *reinterpret_cast<const float4*>(ra + u * kTP + p);
          B4[u] = *reinterpret_cast<const float4*>(rb + u * kTP + p);
        }
#pragma unroll
        for (int u = 0; u < 4; ++u)
#pragma unroll
          for (int v = 0; v < 4; ++v)
            h[u][v] += A4[u].x * B4[v].x + A4[u].y * B4[v].y + A4[u].z * B4[v].z + A4[u].w * B4[v].w;
      }
#pragma unroll
      for (int u = 0; u < 4; ++u)
#pragma unroll
        for (int v = 0; v < 4; ++v) {
          const int r = 4 * bi + u, c = 4 * bj + v;
          if (c >= r && c < kMaxCode + 7) accp[tri_index(r, c)] = h[u][v];
        }
    } else if (tid < 171 + kMaxCode + 7) {
      const int c = tid - 171;
      const float* rj = S.act + c * kTP;
      float s = 0.f;
      for (int p = 0; p < kTP; ++p) s = fmaf(rj[p], S.rr[p], s);
      accp[kAccB + c] = s;
    } else if (tid == 255) {
      float s = 0.f, n = 0.f;
      for (int p = 0; p < kTP; ++p) {
        s = fmaf(S.rr[p], S.rr[p], s);
        n += (tmode() == MODE_SDF) ? S.rscale[p] : (p < nrows ? 1.f : 0.f);
      }
      accp[kAccLoss] = s;
      accp[kAccLoss + 1] = n;
    }
    __syncthreads();
  }
}

}  // namespace dspgn
