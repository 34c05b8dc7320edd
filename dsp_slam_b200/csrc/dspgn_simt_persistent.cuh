// The kernels of the fp32 SIMT engine: k_decoder_simt on the per-iteration schedule (one launch per term and iteration)
// and k_simt_persistent on the persistent object-pipelined schedule (DESIGN §4.12, every GN iteration of every object in
// one launch).  Both run the tile simt_tile (dspgn_simt.cuh) on the tiles of the shared tile source (tile_at,
// dspgn_tc.cuh); the persistent kernel starts each work item with the shared prologue of the tensor-core kernels
// (mega_item_begin) at simt_rows(H) rows per tile.
//
// k_simt_persistent has no producer warpgroup: thread 0 of the CTA pops the next work item into the CTA-local FIFO
// between tiles, behind the barriers that end the previous tile, so the CTA holds no queue ticket while it runs a tile.
// The scan items and the solve step run on the CTA's 256 threads (named barrier 1, as on the 256 epilogue threads of the
// tensor-core kernels).
#pragma once
#include "dspgn_tc.cuh"

namespace dspgn {

// Shared memory of k_simt_persistent: the SIMT tile, then the persistent schedule's state.  The solve workspace and the range words of a ray-sample or band tile both overlay the activation buffer, dead between
// tiles: a tile first writes it after the barrier that ends its phase 0, the last reader of the range words.
template <int H>
struct SimtMegaSmem : SimtSmem<H> {
  MegaSmem mega;
  __device__ SolveSmem& solve_smem() { return *reinterpret_cast<SolveSmem*>(this->act); }
  __device__ int* range_words() { return reinterpret_cast<int*>(this->act); }
};
static_assert(sizeof(SimtMegaSmem<kHid>) <= 227 * 1024 && sizeof(SimtMegaSmem<kHidWide>) <= 227 * 1024,
              "k_simt_persistent: shared memory exceeds the 227 KB per block of sm_90");
static_assert(sizeof(SolveSmem) <= sizeof(SimtSmem<kHid>::act) && sizeof(SolveSmem) <= sizeof(SimtSmem<kHidWide>::act),
              "k_simt_persistent: the solve workspace overlays the activation buffer");
static_assert(4 * (kScanMaxRays + 1) <= sizeof(SimtSmem<kHid>::act) && 4 * (kScanMaxRays + 1) <= sizeof(SimtSmem<kHidWide>::act) &&
              4 * (kScanMaxRays / kSegRays + 1) <= sizeof(SimtSmem<kHid>::act),
              "k_simt_persistent: a ray-sample / band tile stages its object's range words in the activation buffer");

// H: the widest layer of any class of the solver (kHid or kHidWide); every class runs at that instantiation
template <int H>
__global__ void __launch_bounds__(kThreads, 1) k_decoder_simt(BatchDev b, TermArgs a) {
  constexpr int kTP = simt_rows(H);
  extern __shared__ __align__(16) unsigned char smem_raw[];
  SimtSmem<H>& S = *reinterpret_cast<SimtSmem<H>*>(smem_raw);
  build_tile_prefix(b, a, kTP, S.prefix, S.warp_tmp);
  for (int seq = 0;; ++seq) {
    TileRef tr;
    if (!tile_at<kTP, 0>(b, a, S, seq, tr)) break;
    // (the previous tile ended with a barrier of all threads, after its last read of S.obj)
    stage_obj(S.obj, b.state[tr.o], b.decs[b.meta[tr.o].class_id].L, threadIdx.x);
    __syncthreads();
    simt_tile<H, false>(S, b, a, tr.o, tr.row0, tr.slot, tr.mode, SimtMegaTile{});
  }
}

// One CTA per SM (grid_sms); the LayerNorm scratch (a.ln_scratch) holds one region per CTA.
template <int H>
__global__ void __launch_bounds__(kThreads, 1) k_simt_persistent(BatchDev b, TermArgs a, MegaArgs q, SolveArgs sv) {
  constexpr int kTP = simt_rows(H);
  extern __shared__ __align__(16) unsigned char smem_raw[];
  SimtMegaSmem<H>& S = *reinterpret_cast<SimtMegaSmem<H>*>(smem_raw);
  const int tid = threadIdx.x;
  if (tid == 0) S.mega.init(b, q, sv);
  __syncthreads();
  for (int seq = 0;; ++seq) {
    // the previous item ended with a barrier of all threads: take the next one (at most one FIFO entry is ever ahead)
    if (tid == 0) {
      *reinterpret_cast<volatile int*>(&S.mega.epi_seq) = seq;
      mega_fifo_fill(q, b.n_obj, S.mega, seq);
    }
    TileRef tr;
    if (!tile_at<kTP, 2>(b, a, S, seq, tr)) break;
    SimtMegaTile mt{};
    // (publishes seq again: the scheduler is thread 0 itself, which pops item seq + 1 only after this item's barriers)
    if (!mega_item_begin<kTP>(S, b, a, q, sv, tr, seq, tid, mt.iter, mt.term_rows)) continue;
    const int o = tr.o, mode = tr.mode;
    const ObjMeta& M = b.meta[o];
    mt.segp = S.range_words();
    mt.nseg = mega_stage_ranges(q, M, o, mode, S.range_words(), tid, mt.compact);
    mt.seg_samples = kSegRays * b.D;
    __syncthreads();
    simt_tile<H, true>(S, b, a, o, tr.row0, tr.slot, mode, mt);
    mega_tile_end<true, kTP>(S, q, M, o, mode, tr.tile, tid);
  }
}

inline int simt_setup_kernels(int hid, std::string& err) {
  const cudaError_t e = (hid == kHid)
      ? cudaFuncSetAttribute(k_simt_persistent<kHid>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(SimtMegaSmem<kHid>))
      : cudaFuncSetAttribute(k_simt_persistent<kHidWide>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(SimtMegaSmem<kHidWide>));
  if (e != cudaSuccess) {
    err = std::string("cudaFuncSetAttribute(k_simt_persistent): ") + cudaGetErrorString(cudaGetLastError());
    return DSPGN_E_CUDA;
  }
  return 0;
}

}  // namespace dspgn
