// Tensor-core engine for plain decoders up to 512 wide (DSPGN_ENGINE_TC_WIDE), per-iteration schedule, sm_90a.
//
// The 128-row tile of dspgn_tc.cuh cannot be widened to N = 512: its accumulator (64 x 256 fp32 per warpgroup) already
// takes 128 registers per thread and its register-resident hi operand would take another 128 at K = 512.  This tile
// has 64 rows and splits every layer by output column instead of by row:
//
//   * consumer warpgroup g (warps 4g .. 4g+3) owns output columns [256g, 256g + 256) of every GEMM step for all 64 rows
//     of the tile; its accumulator is the same m64n256 fragment as in dspgn_tc.cuh.  In a step with at most 256
//     outputs only warpgroup 0's columns are real (tcw_gemm);
//   * the A operand of a step, hi and lo fp16 halves of the activations (or gradients), lives in shared memory as two
//     128B-swizzled K-major images of 64 rows x 512 K (64 KB each), and both warpgroups read it through descriptors
//     (Wgmma<256>::ss).  Each epilogue writes the next operand in place, after both warpgroups retired the step's MMAs;
//   * weights are packed by tc_pack_images at wgmma N = 256 or 512 rows, so one ring stage (32 K x 512 rows, 32 KB) holds
//     both warpgroups' B operands, 16 KB apart.  One producer lane streams them through a 2-stage ring (produce_step);
//   * layer 0 is a GEMM step of its own (A = [z | x | 0], K = 128): the folded bias ObjState.zb0 of the 256-wide engine
//     has 256 entries, and the per-iteration schedule has no solve step that could refresh a wider one;
//   * ReLU masks go to a per-CTA global scratch ([CTA][layer][consumer thread] of uint4), as in k_gn_persistent; the
//     final Linear(width, 1) + tanh is a per-row dot product, its two column halves combined through shared memory.
//
// Every product is  A_hi W_hi + A_lo W_hi + A_hi W_lo  (fp32 accumulate) as in dspgn_tc.cuh.  The tile writes the
// per-tile partial sums k_solve reads (kAccStride per tile), so everything downstream of launch_term is shared with the
// other engines.  Shared memory: ring 64 KB | A hi 64 KB | A lo 64 KB | TcwSmemTail (J tile, per-row values, plans).
#pragma once
#include <type_traits>
#include "dspgn_tc.cuh"

namespace dspgn {

constexpr int kTcwRows = 64;              // rows per tile
constexpr int kTcwHid = 512;              // widest layer
constexpr int kTcwRing = 2;               // weight ring stages
constexpr int kTcwStageBytes = 32768;     // one stage: 32 K x up to 512 rows x fp16 (64 B rows, SWIZZLE_64B)
constexpr int kTcwAImgBytes = 65536;      // one A image (hi or lo): 8 K chunks x (64 rows x 128 B), SWIZZLE_128B
constexpr int kTcwMaskLayers = 8;         // hidden layers with a saved ReLU mask (nl <= 9)

// weight images and step plan of one decoder class (a solver-owned device array, one entry per class)
struct TcwDecDev {
  const unsigned char* blob;
  TcPlan plan;
};

template <int SCHED>
struct TcwSmemTail {
  float Jp[kTcwRows * kJpStride];         // [row][72+4]: J row of each point; cols 0..66 double as latent_in skip gradient
  float bias[kTcwHid];                    // bias of the current forward step, zero padded
  // object-frame point of every row, x / y / z kTcRows apart (the layout epi_concat_input reads; rows >= 64 unused)
  float xr[3 * kTcRows];
  // per-row values the tail reads (kept here, not in registers, through the step loop): row weight, decoder output,
  // band-row residual
  float rr[kTcwRows], rsc[kTcwRows], scr[kTcwRows], yrow[kTcwRows], rin[kTcwRows];
  float ypart[2 * kTcwRows];              // last layer: each warpgroup's half of the per-row dot product
  TileObj obj;                            // the tile's object (stage_obj)
  int prefix[SCHED == 0 ? kMaxObjScan + 1 : 1];   // tile prefix of the per-iteration schedule (unused by SCHED 1)
  int warp_tmp[32];
  // the tile being run: CTA sequence number, partial-sum slot, object, first row, rows, class.  The step loop and the
  // tail read them from here after each barrier: held in registers through the epilogues, such tile-wide scalars spill
  // to local memory.
  int t_seq, t_tile, t_o, t_row0, t_nrows, t_cls;
  uint64_t w_full[kTcwRing], w_empty[kTcwRing];
  TcPlan plans[DSPGN_MAX_CLASSES];
};
// The persistent kernel's tail (k_wide_persistent): the same fields, then the tile's kind and index in its term and the
// persistent schedule's state.  Its solve workspace is the A hi image and the range words of a ray-sample or band tile's
// object are staged in the A lo image: both images are dead between tiles (the last GEMM step of a tile retired every MMA
// that read them).
struct TcwMegaTail : TcwSmemTail<1> {
  int t_mode, t_j;
  MegaSmem mega;
  __device__ SolveSmem& solve_smem() {
    return *reinterpret_cast<SolveSmem*>(reinterpret_cast<unsigned char*>(this) - 2 * (size_t)kTcwAImgBytes);
  }
};
template <int SCHED> using TcwTail = std::conditional_t<SCHED == 0, TcwSmemTail<0>, TcwMegaTail>;
template <int SCHED>
constexpr size_t kTcwSmemBytesOf = 1024 + (size_t)kTcwRing * kTcwStageBytes + 2 * (size_t)kTcwAImgBytes + sizeof(TcwTail<SCHED>);
constexpr size_t kTcwSmemBytes = kTcwSmemBytesOf<0>, kTcwMegaSmemBytes = kTcwSmemBytesOf<1>;
static_assert(kTcwSmemBytes <= 227 * 1024, "k_wide_wgmma: shared memory exceeds the 227 KB per block of sm_90");
static_assert(kTcwMegaSmemBytes <= 227 * 1024, "k_wide_persistent: shared memory exceeds the 227 KB per block of sm_90");
static_assert(offsetof(TcwSmemTail<0>, bias) % 8 == 0 && offsetof(TcwSmemTail<1>, bias) % 8 == 0,
              "epi_fwd_hidden reads bias column pairs as float2");
static_assert(sizeof(SolveSmem) <= kTcwAImgBytes, "k_wide_persistent: the solve workspace overlays the A hi image");
static_assert(4 * (kScanMaxRays + 1) <= kTcwAImgBytes && 4 * (kScanMaxRays / kSegRays + 1) <= kTcwAImgBytes,
              "k_wide_persistent: a ray-sample / band tile stages its object's range words in the A lo image");

// accumulator-shaped values of warpgroup grp (columns [256 grp, 256 grp + 256)) -> hi / lo A images of the next step
__device__ __forceinline__ void tcw_store_operand(const float (&v)[128], unsigned char* ahi, unsigned char* alo, int rl, int q,
                                                  int grp) {
#pragma unroll
  for (int t = 0; t < 16; ++t) {
#pragma unroll
    for (int h = 0; h < 4; ++h) {       // h: (rows rl / rl+8) x (columns 16t+2q / 16t+8+2q)
      uint32_t hi, lo;
      split_pack(v[8 * t + 2 * h], v[8 * t + 2 * h + 1], hi, lo);
      const int row = rl + 8 * (h & 1), kk = 256 * grp + 16 * t + 8 * (h >> 1) + 2 * q;
      const int off = (kk >> 6) * 8192 + row * 128 + ((((kk & 63) >> 3) ^ (row & 7)) << 4) + (kk & 7) * 2;
      *reinterpret_cast<uint32_t*>(ahi + off) = hi;
      *reinterpret_cast<uint32_t*>(alo + off) = lo;
    }
  }
}

// One GEMM step of warpgroup grp: acc = A * W^T over nch K chunks of 64, A hi / lo from the shared images, W through the
// 2-stage ring.  The stages of a chunk arrive as hi[k 0..31], hi[k 32..63], lo[k 0..31], lo[k 32..63] (tc_pack_images),
// so every output accumulates  A_hi W_hi, A_lo W_hi  per K-step, then  A_hi W_lo.  Behind each stage `wait_group 1`
// retires the previous stage's MMAs and that stage goes back to the producer.  In a step with at most 256 outputs
// warpgroup 1 multiplies whatever the upper half of the stage holds: its columns are >= the step's n_real, and every
// epilogue selects 0 (or the decoder input) there without reading them.  Skipping its MMAs instead puts the wgmma
// sequence under a branch ptxas cannot prove uniform, and it serializes every wgmma of the kernel (C7518).
__device__ __forceinline__ void tcw_gemm(float (&acc)[128], uint32_t ahi, uint32_t alo, uint32_t ring_g, uint32_t bars,
                                         uint32_t& stage, uint32_t& phase, int nch) {
  const uint32_t w_full = bars, w_empty = bars + 8u * kTcwRing;
#pragma unroll
  for (int i = 0; i < 128; ++i) acc[i] = 0.f;
  uint32_t prev = 0;
  for (int c = 0; c < nch; ++c) {
#pragma unroll
    for (int s = 0; s < kTcStages; ++s) {
      uint32_t slot, ph;
      ring_at<kTcwRing>(stage, phase, (uint32_t)(kTcStages * c + s), slot, ph);
      mbar_wait(w_full + 8u * slot, ph);
      wg_fence();
      const uint32_t bw = ring_g + slot * kTcwStageBytes;
#pragma unroll
      for (int k = 0; k < 2; ++k) {
        const uint32_t ao = 8192u * (uint32_t)c + 32u * (uint32_t)(2 * (s & 1) + k);
        const uint64_t bd = make_desc_w(bw + 32u * k);
        // columns >= the step's n_real (stale ring bytes for warpgroup 1 on a narrow step) must never reach an epilogue
        // read: every epi_* pass selects 0 or the decoder input there
        Wgmma<256>::ss(acc, make_desc(ahi + ao), bd);
        if (s < 2) Wgmma<256>::ss(acc, make_desc(alo + ao), bd);
      }
      wg_commit();
      wg_wait1();
      if (c > 0 || s > 0) release_stage(w_empty, (int)prev);
      prev = slot;
    }
  }
  wg_wait0();
  release_stage(w_empty, (int)prev);
  ring_at<kTcwRing>(stage, phase, (uint32_t)(kTcStages * nch), stage, phase);
}

// The wide tile loop of both schedules.  SCHED 0 (k_wide_wgmma): one launch per term and iteration, static round-robin
// over the launch's tiles (a.mode is the tile kind).  SCHED 1 (k_wide_persistent): every GN iteration of every object
// in one launch, the work items of the device queue (ray-sample, scan, band and SDF items at kTcwRows rows per tile)
// through the CTA-local FIFO, the solve step and the next iteration's items in the CTA that finishes an object's
// iteration -- the scheduling of k_gn_persistent_render (dspgn_tc.cuh: mega_*), with this tile.
template <int SCHED>
__device__ __forceinline__ void tcw_body(const BatchDev& b, const TermArgs& a, const TcwDecDev* __restrict__ wd,
                                         uint4* __restrict__ masks_g, const MegaArgs& q, const SolveArgs& sv) {
  constexpr bool MEGA = SCHED == 1;
  constexpr int SRC = MEGA ? 2 : 0;             // tile_at: static tiles, or every item kind from the FIFO
  extern __shared__ unsigned char tcw_smem_raw[];
  unsigned char* ring = tcw_smem_raw + ((1024u - (smem_u32(tcw_smem_raw) & 1023u)) & 1023u);
  unsigned char* const ahi = ring + (size_t)kTcwRing * kTcwStageBytes;
  unsigned char* const alo = ahi + kTcwAImgBytes;
  TcwTail<SCHED>& S = *reinterpret_cast<TcwTail<SCHED>*>(alo + kTcwAImgBytes);
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;

  if (!MEGA) build_tile_prefix(b, a, kTcwRows, S.prefix, S.warp_tmp);
  stage_plans(S.plans, b.n_classes, [&](int c) -> const TcPlan& { return wd[c].plan; }, tid);
  if (tid == 0) {
    for (int i = 0; i < kTcwRing; ++i) { mbar_init(&S.w_full[i], 1); mbar_init(&S.w_empty[i], 8); }
    if constexpr (MEGA) S.mega.init(b, q, sv);
    fence_barrier_init();
  }
  __syncthreads();

  if (warp >= 8) {
    // ===================== weight producer (warp 8 lane 0; SCHED 1: also the CTA's scheduler) =================
    setmaxnreg_dec<kTcProducerRegs>();
    if (warp == 8 && lane == 0) {
      uint32_t stage = 0, phase = 0;
      for (int seq = 0;; ++seq) {
        if constexpr (MEGA) mega_fifo_fill(q, b.n_obj, S.mega, seq);
        TileRef tr;
        if (!tile_at<kTcwRows, SRC>(b, a, S, seq, tr)) break;
        const int cls = b.meta[tr.o].class_id;
        produce_tile<kTcwRing, kTcwStageBytes>(wd[cls].blob, S.plans[cls], tile_steps<MEGA>(S.plans[cls], tr.mode), ring, S.w_full,
                                               S.w_empty, stage, phase);
      }
    }
    return;
  }
  // ===================== consumer warpgroups =====================================================
  setmaxnreg_inc<kTcConsumerRegs>();
  const int grp = warp >> 2;
  // per-row stages: thread = tile row (4 copies, tid < 64 writes); read afresh from %tid.x where used, not kept live
  auto tile_row = [] { uint32_t t; asm volatile("mov.u32 %0, %%tid.x;" : "=r"(t)); return (int)(t & (kTcwRows - 1)); };
  const int qd = lane & 3;
  const int rl = 16 * (warp & 3) + (lane >> 2);              // fragment rows rl, rl + 8
  const int rowA = rl, rowB = rl + 8;
  const uint32_t ahi_s = smem_u32(ahi), alo_s = smem_u32(alo);
  const uint32_t ring_g = smem_u32(ring) + (uint32_t)grp * (kTcwStageBytes / 2);
  const uint32_t bars = smem_u32(S.w_full);
  // SCHED 0: the launch's term; SCHED 1: the tile's kind, read from S.t_mode where it is needed
  const int mode0 = a.mode;
  const bool grid_mode = !MEGA && mode0 == MODE_GRIDFWD;
  const bool fwd_only0 = mode0 == MODE_RAYFWD || mode0 == MODE_PTSFWD || grid_mode;
  const bool pts_mode0 = mode0 == MODE_SDF || mode0 == MODE_PTSFWD || grid_mode;
  auto tile_mode = [&] { if constexpr (MEGA) return *reinterpret_cast<volatile int*>(&S.t_mode); else return mode0; };
  uint32_t stage = 0, phase = 0;
  float acc[128];
  // The sequence number, the tile count (S.prefix[n_obj]) and this thread's tile row are read from shared memory / %tid
  // where they are needed, so that nothing tile-wide stays in registers through the epilogues.
  for (int seq = 0;; ++seq) {
    // ---- prologue: the object's pose, code and this row's point --------------------------------------------------
    {
      TileRef tr;
      if (!tile_at<kTcwRows, SRC>(b, a, S, seq, tr)) break;
      int iter = a.iter, term_n = 0;
      if constexpr (MEGA) {
        if (!mega_item_begin<kTcwRows>(S, b, a, q, sv, tr, seq + 1, tid, iter, term_n)) continue;
        if (tid == 0) { S.t_mode = tr.mode; S.t_j = tr.tile; }
      } else {
        stage_obj(S.obj, b.state[tr.o], b.decs[b.meta[tr.o].class_id].L, tid);
        term_n = term_rows(b, a, tr.o);
      }
      const int o = tr.o, row0 = tr.row0, mode = tr.mode;
      const bool pts_mode = MEGA ? mode == MODE_SDF : pts_mode0;
      const ObjMeta& M = b.meta[o];
      const ObjState& ost = b.state[o];
      const int L = b.decs[M.class_id].L;
      const uint8_t* mask_in; uint8_t* mask_out;
      cut_masks(a, ost.mode, iter, mask_in, mask_out);
      const int nrows = min(kTcwRows, term_n - row0);
      // SCHED 1: the object's range words for the row -> sample map of a ray-sample or band tile, in the dead A lo image
      const int* segp = reinterpret_cast<const int*>(alo);
      bool compact = false;
      const int nseg = MEGA ? mega_stage_ranges(q, M, o, mode, reinterpret_cast<int*>(alo), tid, compact) : 0;
      epi_bar_sync();      // the previous tile's per-row stages are done with xr / scr and the tile descriptor
      const int r = tile_row();
      if (tid == 0) { S.t_seq = seq; S.t_tile = tr.slot; S.t_o = o; S.t_row0 = row0; S.t_nrows = nrows; S.t_cls = M.class_id; }
      float x0 = 0.f, x1 = 0.f, x2 = 0.f, res_in = 0.f, sc = 0.f;
      if (r < nrows) {
        const int rr_ = row0 + r;
        if (pts_mode) {
          const float* pq = grid_mode ? a.grid + 3 * (size_t)rr_ : b.pts + 3 * (size_t)(M.pts_off + rr_);
          if (grid_mode) { x0 = pq[0]; x1 = pq[1]; x2 = pq[2]; }
          else xform_point(S.obj.ost, pq[0], pq[1], pq[2], x0, x1, x2);
          sc = (grid_mode || mask_in == nullptr || ldv(mask_in + M.pts_off + rr_)) ? 1.f : 0.f;
        } else if (mode == MODE_BAND) {
          const size_t sidx = MEGA ? band_row_sample(segp, nseg, M.smp_off, (size_t)kSegRays * b.D, rr_) : (size_t)M.smp_off + rr_;
          x0 = __ldcg(b.band_x + 3 * sidx); x1 = __ldcg(b.band_x + 3 * sidx + 1); x2 = __ldcg(b.band_x + 3 * sidx + 2);
          sc = __ldcg(b.band_s + sidx); res_in = __ldcg(b.band_r + sidx);
        } else {
          sc = ray_sample_row(b, M, S.obj.ost, S.obj.ost[12], S.obj.ost[13], S.obj.ost[14], segp, compact, rr_, x0, x1, x2);
        }
      }
      if (tid < kTcwRows) { S.xr[r] = x0; S.xr[kTcRows + r] = x1; S.xr[2 * kTcRows + r] = x2; S.scr[r] = sc; S.rin[r] = res_in; }
      epi_bar_sync();
      // ---- A operand of the first GEMM step (layer 0): the decoder input [z | x | 0...], K = 16 k_steps ---------------
      const int kh = S.plans[M.class_id].step[0].k_steps * 8;            // column pairs per row
      for (int i = tid; i < kTcwRows * kh; i += kTcEpiThreads) {
        const int row = i / kh, kk = 2 * (i - row * kh);
        float v[2];
#pragma unroll
        for (int u = 0; u < 2; ++u) {
          const int j = kk + u - L;
          v[u] = (j < 0) ? S.obj.zs[kk + u] : ((unsigned)j < 3u ? S.xr[j * kTcRows + row] : 0.f);
        }
        uint32_t hi, lo;
        split_pack(v[0], v[1], hi, lo);
        const int off = (kk >> 6) * 8192 + row * 128 + ((((kk & 63) >> 3) ^ (row & 7)) << 4) + (kk & 7) * 2;
        *reinterpret_cast<uint32_t*>(ahi + off) = hi;
        *reinterpret_cast<uint32_t*>(alo + off) = lo;
      }
      fence_proxy_async();
      epi_bar_sync();
    }
    // this thread's ReLU masks, layer l at mg[l * 256].  Only tiles with a backward chain touch the scratch: the
    // forward-only ray-sample pass runs beside the SDF-row pass on a second stream, with the same CTA indices.
    uint4* const mg = masks_g + (size_t)blockIdx.x * kTcwMaskLayers * kTcEpiThreads + tid;
    for (int s = 0;; ++s) {
      const int cls = S.t_cls;
      const TcPlan& plan = S.plans[cls];
      const bool fwd_only = MEGA ? tile_mode() == MODE_RAYFWD : fwd_only0;
      const int ns = tile_steps<MEGA>(plan, tile_mode());
      if (s >= ns) break;
      const DecoderDev& dec = b.decs[cls];
      const TcStep st = plan.step[s];
      const bool more = s + 1 < ns;
      const int k_next = more ? plan.step[s + 1].k_steps * 16 : 0;
      const int nm = st.n_real;
      if constexpr (MEGA) { if (tid == 0 && s == 0) log_event(q.log, ev_desc(EV_FIRST_MMA, tile_mode(), S.t_o, S.t_j)); }
      // a forward step's bias, read by its epilogue after the barrier below (the previous epilogue's reads ended
      // before the barrier that published this step's operand)
      if (st.kind == TK_FWD_HIDDEN || st.kind == TK_FWD_PENULT) {
        const float* bg = dec.bias[st.layer];
        for (int i = tid; i < kTcwHid; i += kTcEpiThreads) S.bias[i] = (i < nm) ? __ldg(bg + i) : 0.f;
      }
      tcw_gemm(acc, ahi_s, alo_s, ring_g, bars, stage, phase, st.k_steps / 4);
      epi_bar_sync();                                  // both warpgroups have retired their MMAs: the A images are free
      const int qs = opaque_int(qd);
      const int c0 = 256 * grp;
      bool store = more;
      if (st.kind == TK_FWD_PENULT) {
        // ---- last hidden layer: bias + ReLU (mask saved), then Linear(width, 1) + tanh as a per-row dot product
        // (deep_sdf_decoder.py:91,103,107-108): each warpgroup's half over its quad, the halves through shared memory
        float pa = 0.f, pb = 0.f;
        uint32_t mw[4] = {0u, 0u, 0u, 0u};
#pragma unroll
        for (int e = 0; e < 128; ++e) {
          const int c = c0 + frag_col(e, qs);
          if (c < nm) {
            const float w = acc[e] + S.bias[c];
            mw[e >> 5] |= (w > 0.f ? 1u : 0u) << (e & 31);
            if (e & 2) pb = fmaf(fmaxf(w, 0.f), __ldg(dec.w_last + c), pb);
            else pa = fmaf(fmaxf(w, 0.f), __ldg(dec.w_last + c), pa);
          }
        }
        if (!fwd_only) mg[st.layer * kTcEpiThreads] = make_uint4(mw[0], mw[1], mw[2], mw[3]);
        pa += __shfl_xor_sync(0xffffffffu, pa, 1);
        pb += __shfl_xor_sync(0xffffffffu, pb, 1);
        pa += __shfl_xor_sync(0xffffffffu, pa, 2);
        pb += __shfl_xor_sync(0xffffffffu, pb, 2);
        if (qd == 0) { S.ypart[grp * kTcwRows + rowA] = pa; S.ypart[grp * kTcwRows + rowB] = pb; }
        epi_bar_sync();
        if (tid < kTcwRows) S.yrow[tid] = tanhf(S.ypart[tid] + S.ypart[kTcwRows + tid] + __ldg(dec.bias[st.layer + 1]));
        epi_bar_sync();
        if (fwd_only) {
          const int r = tile_row();
          const float sc = S.scr[r];
          const int o = S.t_o, row0 = S.t_row0, nrows = S.t_nrows;
          const ObjMeta& M = b.meta[o];
          const int mode = tile_mode();
          if (tid < kTcwRows && r < nrows) {
            const size_t base = (mode == MODE_RAYFWD) ? (size_t)M.smp_off
                                : (grid_mode ? (size_t)a.grid_slot[o] * a.grid_rows : (size_t)M.pts_off);
            b.sdf[base + row0 + r] = (sc != 0.f) ? S.yrow[r] : INFINITY;
          }
          if (!MEGA && mode == MODE_RAYFWD) {          // (persistent kernel: counted by the scan items, scan_chunk)
            const unsigned bal = __ballot_sync(0xffffffffu, tid < kTcwRows && r < nrows && sc != 0.f);
            if (lane == 0 && bal) atomicAdd(b.V_count + o, __popc(bal));
          }
        }
        if (more) {
          // seed of the backward chain: g = (1 - y^2) W_last, masked by this layer's ReLU
          const float ya = S.yrow[rowA], yb = S.yrow[rowB];
          const float ga = 1.f - ya * ya, gb = 1.f - yb * yb;
#pragma unroll
          for (int e = 0; e < 128; ++e) {
            const int c = c0 + frag_col(e, qs);
            acc[e] = ((mw[e >> 5] >> (e & 31)) & 1u) ? ((e & 2) ? gb : ga) * __ldg(dec.w_last + c) : 0.f;
          }
        }
      } else if (st.kind == TK_FWD_HIDDEN) {
        // the epi_* passes of tc_body on this warpgroup's columns: bounds and the concat offset relative to c0
        uint32_t mw[4] = {0u, 0u, 0u, 0u};
        epi_fwd_hidden<0, 0>(acc, mw, S.bias + c0, qs, nm - c0, k_next - c0);
        if (st.cat_off >= 0) epi_concat_input<0, 0>(acc, qs, k_next - c0, st.cat_off - c0, dec.L, S.obj.zs, S.xr, rowA, rowB);
        if (!fwd_only) mg[st.layer * kTcEpiThreads] = make_uint4(mw[0], mw[1], mw[2], mw[3]);
      } else if (st.kind == TK_BWD_MID) {
        const uint4 m4 = mg[st.mask_layer * kTcEpiThreads];
        const uint32_t mw[4] = {m4.x, m4.y, m4.z, m4.w};
        if (st.cat_off >= 0) epi_skip_grad<0, 0>(acc, qs, nm - c0, st.cat_off - c0, dec.in0, dec.L, S.Jp, rowA, rowB);
        epi_bwd_mid<0, 0>(acc, mw, nm - c0, k_next - c0);
      } else {
        // ---- TK_BWD_FIRST: d/d(input) complete -> Jacobian row; its in0 <= 80 columns are all warpgroup 0's
        if (grp == 0) epi_bwd_first(acc, qs, dec.in0, dec.L, dec.latent_in >= 0, S.Jp, S.scr, rowA, rowB);
        store = false;
      }
      if (store) {
        tcw_store_operand(acc, ahi, alo, rl, qd, grp);
        fence_proxy_async();
        epi_bar_sync();
      }
    }
    // (the tile descriptor is rewritten after the first barrier of the next tile's prologue)
    if (MEGA ? tile_mode() == MODE_RAYFWD : fwd_only0) {
      seq = S.t_seq;
      if constexpr (MEGA) mega_tile_end<true, kTcwRows>(S, q, b.meta[S.t_o], S.t_o, MODE_RAYFWD, S.t_j, tid);
      continue;
    }
    // ---- pose columns, residual (thread = row; needs every d/d(input) column of the row) -----------------------------
    epi_bar_sync();
    const int o = S.t_o, row0 = S.t_row0, nrows = S.t_nrows, r = tile_row();
    const ObjState& ost = b.state[o];
    const int mode = tile_mode();
    if (tid < kTcwRows) {
      const int L = b.decs[S.t_cls].L;
      const uint8_t* mask_in; uint8_t* mask_out;
      cut_masks(a, ost.mode, (MEGA && a.cut_iter >= 0) ? ldv(q.obj_iter + o) : a.iter, mask_in, mask_out);
      const float huber_b = term_huber(a, mode, ost.mode, (MEGA && mode == MODE_BAND) ? a.huber_b1 : a.huber_b);
      float* jr = S.Jp + r * kJpStride;
      for (int i = L; i < kMaxCode; ++i) jr[i] = 0.f;
      const RowTail t = row_tail(jr, 1, S.xr[r], S.xr[kTcRows + r], S.xr[2 * kTcRows + r], jr[kMaxCode], jr[kMaxCode + 1],
                                 jr[kMaxCode + 2], (mode == MODE_SDF) ? S.yrow[r] : S.rin[r], S.scr[r], r, nrows, mode,
                                 ost.mode, huber_b, mask_out, b.meta[o].pts_off + row0);
      S.rr[r] = t.rho_r;
      jr[kMaxCode + 7] = t.rho_r;                       // for jtile_sums: J^T (rho r) from the J^T J chains
      S.rsc[r] = t.n;
      if (a.dbg_J != nullptr && o == a.dbg_obj && mode == MODE_SDF && r < nrows) a.dbg_res[row0 + r] = t.res;
    }
    epi_bar_sync();
    if (a.dbg_J != nullptr && o == a.dbg_obj && mode == MODE_SDF)
      dbg_dump_J(a, S.Jp, kJpStride, 1, row0, nrows, ost.mode, tid, kTcEpiThreads);
    jtile_sums<kTcwRows>(S.Jp, S.rr, S.rsc, ((MEGA && mode == MODE_BAND) ? a.part_r : a.part) + (size_t)S.t_tile * kAccStride, tid);
    seq = S.t_seq;
    // the next tile's prologue starts with epi_bar_sync(): Jp / rr are not rewritten before it
    if constexpr (MEGA) mega_tile_end<true, kTcwRows>(S, q, b.meta[o], o, mode, S.t_j, tid);
  }
}

__global__ void __launch_bounds__(kTcThreads, 1) k_wide_wgmma(BatchDev b, TermArgs a, const TcwDecDev* __restrict__ wd,
                                                               uint4* __restrict__ masks_g) {
  tcw_body<0>(b, a, wd, masks_g, MegaArgs{}, SolveArgs{});
}
// Persistent object-pipelined variant: all GN iterations of all objects in ONE launch, every item kind (SDF-only and
// pose-only runs simply queue no ray-sample items).  masks: the ReLU mask scratch, as for k_wide_wgmma.
__global__ void __launch_bounds__(kTcThreads, 1) k_wide_persistent(BatchDev b, TermArgs a, MegaArgs q, SolveArgs sv,
                                                                       const TcwDecDev* __restrict__ wd, uint4* __restrict__ masks) {
  tcw_body<1>(b, a, wd, masks, q, sv);
}

// ------------------------------------------------------------------------------------------------
// host side: plan + weight images
// ------------------------------------------------------------------------------------------------
// wgmma N of a step with n outputs: warpgroup 0 alone (256) or both (512)
constexpr int tcw_mma_n(int n) { return n <= 256 ? 256 : 512; }

// Step plan and weight images of a plain decoder (at most one latent_in layer among the hidden layers, nothing else)
// with layers up to 512 wide.  W[k]: row-major [out_dim][in_dim] of layer k.  Forward steps k = 0 .. nl-2 (layer 0
// included: A = the decoder input), backward steps k = nl-2 .. 0; the final Linear(width, 1) is no step.  Returns false
// for a decoder outside the shape.
inline bool tcw_shape_ok(const DecoderDev& dv) {
  const int nl = dv.n_lin;
  if (dv.generic || nl < 2 || nl - 1 > kTcwMaskLayers || dv.in0 > 80) return false;   // in0 <= 80: epi_bwd_first
  for (int k = 0; k < nl; ++k)
    if (dv.in_dim[k] > kTcwHid || dv.out_dim[k] > kTcwHid) return false;
  return true;
}

inline bool tcw_plan_decoder(const DecoderDev& dv, const float* const* W, TcPlan& P, std::vector<unsigned char>& blob) {
  const int nl = dv.n_lin, li = dv.latent_in, in0 = dv.in0;
  memset(&P, 0, sizeof(TcPlan));
  blob.clear();
  if (!tcw_shape_ok(dv)) return false;
  int ns = 0;
  for (int k = 0; k < nl - 1; ++k) {
    TcStep& s = P.step[ns++];
    const int nin = dv.in_dim[k], nout = dv.out_dim[k];
    s.kind = (k == nl - 2) ? TK_FWD_PENULT : TK_FWD_HIDDEN;
    s.n_mma = tcw_mma_n(nout);
    s.k_steps = tc_pad_k_steps(round16(nin) / 16);
    s.layer = k; s.n_real = nout;
    s.cat_off = (k + 1 == li) ? nout : -1;
    s.mask_layer = -1;
    s.w_off = (unsigned)blob.size();
    const float* Wk = W[k];
    tc_pack_images(blob, s.n_mma, s.k_steps, [&](int n, int kk) { return (n < nout && kk < nin) ? Wk[(size_t)n * nin + kk] : 0.f; });
  }
  P.n_fwd = ns;
  for (int k = nl - 2; k >= 0; --k) {
    TcStep& s = P.step[ns++];
    const int nin = dv.in_dim[k], nout = dv.out_dim[k];
    s.kind = (k == 0) ? TK_BWD_FIRST : TK_BWD_MID;
    s.n_mma = tcw_mma_n(nin);
    s.k_steps = tc_pad_k_steps(round16(nout) / 16);
    s.layer = k; s.n_real = nin;
    s.cat_off = (k == li) ? nin - in0 : -1;
    s.mask_layer = (k > 0) ? k - 1 : -1;
    s.w_off = (unsigned)blob.size();
    const float* Wk = W[k];
    tc_pack_images(blob, s.n_mma, s.k_steps, [&](int n, int kk) { return (n < nin && kk < nout) ? Wk[(size_t)kk * nin + n] : 0.f; });
  }
  P.n_steps = ns;
  return true;
}

// The images of a created decoder, built from its forward weight images on the device (Wf[k][i * H + j] = W_k[j][i]):
// the decoder keeps no host copy of its weights, and only a solver that asks for this engine pays for the blob.
inline int tcw_pack_decoder(const DecoderDev& dv, int H, TcDecoderHost& h, TcPlan& P, std::string& err) {
  h.ok = false;
  if (!tcw_shape_ok(dv)) return 0;
  std::vector<std::vector<float>> w(dv.n_lin);
  std::vector<const float*> W(dv.n_lin);
  for (int k = 0; k < dv.n_lin; ++k) {
    const int nin = dv.in_dim[k], nout = dv.out_dim[k];
    std::vector<float> wf((size_t)nin * H);
    if (cudaMemcpy(wf.data(), dv.Wf[k], wf.size() * sizeof(float), cudaMemcpyDeviceToHost) != cudaSuccess) {
      cudaGetLastError(); err = "cudaMemcpy(decoder weights)"; return DSPGN_E_CUDA;
    }
    w[k].resize((size_t)nout * nin);
    for (int j = 0; j < nout; ++j)
      for (int i = 0; i < nin; ++i) w[k][(size_t)j * nin + i] = wf[(size_t)i * H + j];
    W[k] = w[k].data();
  }
  std::vector<unsigned char> blob;
  if (!tcw_plan_decoder(dv, W.data(), P, blob)) return 0;
  void* d = nullptr;
  if (cudaMalloc(&d, blob.size()) != cudaSuccess) { cudaGetLastError(); err = "cudaMalloc(tc wide blob)"; return DSPGN_E_ALLOC; }
  if (cudaMemcpy(d, blob.data(), blob.size(), cudaMemcpyHostToDevice) != cudaSuccess) { cudaFree(d); err = "cudaMemcpy(tc wide blob)"; return DSPGN_E_CUDA; }
  h.blob = d; h.blob_bytes = blob.size(); h.ok = true;
  return 0;
}

inline int tcw_setup_kernel(std::string& err) {
  if (cudaFuncSetAttribute(k_wide_wgmma, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kTcwSmemBytes) != cudaSuccess) {
    err = std::string("cudaFuncSetAttribute(k_wide_wgmma): ") + cudaGetErrorString(cudaGetLastError());
    return DSPGN_E_CUDA;
  }
  if (cudaFuncSetAttribute(k_wide_persistent, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kTcwMegaSmemBytes) != cudaSuccess) {
    err = std::string("cudaFuncSetAttribute(k_wide_persistent): ") + cudaGetErrorString(cudaGetLastError());
    return DSPGN_E_CUDA;
  }
  return 0;
}

inline void tcw_launch_term(const BatchDev& b, const TermArgs& a, const TcwDecDev* wd, uint4* masks, int grid_max,
                            long long tiles_upper, cudaStream_t stream) {
  int grid = (int)std::min<long long>(tiles_upper, grid_max);
  if (grid < 1) grid = 1;
  k_wide_wgmma<<<grid, kTcThreads, kTcwSmemBytes, stream>>>(b, a, wd, masks);
}

}  // namespace dspgn
