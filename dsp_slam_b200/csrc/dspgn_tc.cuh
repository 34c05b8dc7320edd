// wgmma tensor-core decoder engine for H100 (sm_90a).
//
// One persistent CTA per SM walks 128-row tiles.  For each tile the whole DeepSDF forward chain, the
// backward-to-input chain and the Jacobian / J^T J reduction run without leaving the SM:
//
//   * two consumer warpgroups own 64 tile rows each; their accumulators (64 x 256 fp32) live in registers.  The
//     epilogue works on the accumulator fragment in place: bias/ReLU (forward) or the saved ReLU mask (backward), then
//     every fp32 value is split into fp16 hi + fp16 lo.  The wgmma accumulator fragment of columns [16t, 16t+16) is
//     exactly the register A fragment of K-step t, so the hi halves stay in registers as the next GEMM's A operand and
//     the lo halves go to a 128B-swizzled shared-memory image (A from a descriptor);
//   * weights are pre-split (hi/lo fp16), pre-swizzled (64B swizzle, K-major, 32-wide K halves, padded to the step's
//     wgmma N of 80, 192 or 256 rows) on the host into exactly the shared-memory images the wgmma descriptor expects,
//     and streamed from L2 through a 4 x 16 KB ring with 1-D bulk copies (cp.async.bulk) signalling mbarriers;
//   * every product is formed as  A_hi*W_hi + A_lo*W_hi + A_hi*W_lo  (3 fp16 MMAs, fp32 accumulate):
//     ~2^-21 relative error per product, which keeps the Gauss-Newton iteration inside the fp32 noise
//     floor of the reference (SURVEY.md B.3: >= 15 mantissa bits needed; bf16/tf32 single pass is not);
//   * only the hidden width x width layers are GEMM steps (14 per fwd+bwd tile of the 8 x 256 decoder): layer 0, with
//     its latent part folded into a per-object bias, is 3 FMAs per output while the first operand is built, and the
//     final Linear(width, 1) + tanh is a per-row dot product in the epilogue of the last hidden layer;
//   * J^T J / J^T r of the tile on the CUDA cores, written as per-tile partials.
//
// Warp roles (384 threads): warps 0-3 / 4-7 = consumer warpgroups (MMA issue + epilogue, rows [64g, 64g+64)), warps
// 8-11 = producer warpgroup: warp 8 lane 0 is the weight producer and, in the persistent kernels, the CTA's scheduler
// (pops the device work queue); warps 9-11 exit after giving their registers to the consumers (setmaxnreg).
//
// Three schedules share this body (template SCHED): 0 = one launch per term and iteration (k_decoder_tc), 1 = persistent
// kernel with SDF tiles only (k_gn_persistent), 2 = persistent kernel with the render term: ray-sample tiles (only the run
// of samples inside the unit sphere of every ray: dspgn_solve.cuh, valid_sample_ranges), 64-ray scan items, band tiles,
// SDF tiles (k_gn_persistent_render).  The CTA that completes an object's last outstanding tile runs its solve
// (dspgn_solve.cuh), the next iteration's sample ranges, and queues the next iteration.
//
// Restates the same reference arithmetic as dspgn_simt.cuh (loss.py:22-43,143-150; loss_utils.py:51-103;
// deep_sdf_decoder.py:75-110; optimizer.py:161-167).
#pragma once
#include <cuda_fp16.h>
#include <string>
#include <vector>
#include "dspgn_simt.cuh"
#include "dspgn_solve.cuh"

namespace dspgn {

constexpr int kTcThreads = 384;          // 2 consumer warpgroups + 1 producer warpgroup
constexpr int kTcEpiThreads = 256;
constexpr int kTcStages = 4;              // one 64-wide K chunk: hi[k 0..31], hi[k 32..63], lo[k 0..31], lo[k 32..63]
constexpr int kTcStageBytes = 16384;      // one ring stage: up to 256 rows x 32 K x fp16 (64 B rows, SWIZZLE_64B)
// Stages of the weight ring of a schedule (tc_body SCHED): one K chunk, or one and a half in the SDF-tile kernel, whose
// ReLU masks live in global memory (TcSmemTail) to make room.  Deeper, the ring keeps refills further ahead of the MMAs
// and holds more of the next step while an epilogue runs.
template <int SCHED> constexpr int kTcRing = SCHED == 1 ? 6 : kTcStages;
constexpr int kTcAloBytes = 32768;        // lo halves of one warpgroup's A operand: 4 x (64 rows x 128 B)
// Registers are allocated per warpgroup: the producer warpgroup hands most of its share to the two consumer
// warpgroups (setmaxnreg), which hold the fp32 accumulator (128) and the register A fragment (64).  The pair must fit
// the 384 x 168 registers the launch bound gives the CTA.
constexpr int kTcProducerRegs = 40, kTcConsumerRegs = 232;
static_assert(128 * kTcProducerRegs + 256 * kTcConsumerRegs <= 384 * 168, "setmaxnreg budget exceeds the CTA's registers");

// wgmma N of a GEMM step with `n` output columns: the narrowest instantiated N (80, 192, 256) that holds them.  The
// weight images of the step hold exactly that many rows.
__host__ __device__ constexpr int tc_mma_n(int n) { return n <= 80 ? 80 : (n <= 192 ? 192 : 256); }
// K of every GEMM step is padded to whole 64-wide chunks (zero weight columns): each chunk is one fixed MMA sequence
__host__ __device__ constexpr int tc_pad_k_steps(int k_steps) { return (k_steps + 3) / 4 * 4; }

// ------------------------------------------------------------------------------------------------
// PTX wrappers
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  asm volatile(
      "{\n\t"
      ".reg .pred p;\n\t"
      "WAIT_LOOP:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
      "@p bra DONE;\n\t"
      "bra WAIT_LOOP;\n\t"
      "DONE:\n\t"
      "}" ::"r"(bar), "r"(parity) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) { mbar_wait(smem_u32(bar), parity); }
__device__ __forceinline__ void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }

__device__ __forceinline__ void bulk_g2s(void* smem_dst, const void* gmem_src, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(smem_dst)),
               "l"(gmem_src), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}

// 16 bytes global -> shared, bypassing L1; cp_async_wait_all: every earlier cp_async_16 of this thread has landed
__device__ __forceinline__ void cp_async_16(uint32_t smem_dst, const void* gmem_src) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_dst), "l"(gmem_src) : "memory");
}
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_all;" ::: "memory"); }

// generic-proxy shared-memory writes (the A lo image) before the async proxy (wgmma) reads them
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_wait0() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }
__device__ __forceinline__ void wg_wait1() { asm volatile("wgmma.wait_group.sync.aligned 1;" ::: "memory"); }
template <int REGS> __device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(REGS)); }
template <int REGS> __device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(REGS)); }
// the 128 threads of consumer warpgroup g (ids 1 / 2 are taken by the epilogue and the solve step)
__device__ __forceinline__ void wg_bar_sync(int g) { asm volatile("bar.sync %0, 128;" ::"r"(3 + g) : "memory"); }

#define DSPGN_D8(o) "+f"(d[o + 0]), "+f"(d[o + 1]), "+f"(d[o + 2]), "+f"(d[o + 3]), "+f"(d[o + 4]), "+f"(d[o + 5]), "+f"(d[o + 6]), "+f"(d[o + 7])
#define DSPGN_D128                                                                                                    \
  DSPGN_D8(0), DSPGN_D8(8), DSPGN_D8(16), DSPGN_D8(24), DSPGN_D8(32), DSPGN_D8(40), DSPGN_D8(48), DSPGN_D8(56),         \
      DSPGN_D8(64), DSPGN_D8(72), DSPGN_D8(80), DSPGN_D8(88), DSPGN_D8(96), DSPGN_D8(104), DSPGN_D8(112), DSPGN_D8(120)
#define DSPGN_D96                                                                                                     \
  DSPGN_D8(0), DSPGN_D8(8), DSPGN_D8(16), DSPGN_D8(24), DSPGN_D8(32), DSPGN_D8(40), DSPGN_D8(48), DSPGN_D8(56),         \
      DSPGN_D8(64), DSPGN_D8(72), DSPGN_D8(80), DSPGN_D8(88)
#define DSPGN_D40 DSPGN_D8(0), DSPGN_D8(8), DSPGN_D8(16), DSPGN_D8(24), DSPGN_D8(32)
#define DSPGN_ACC_OPS128 "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, %80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, %96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, %112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127}, "
#define DSPGN_ACC_OPS96 "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, %80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95}, "
#define DSPGN_ACC_OPS40 "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39}, "

// D[64 x N] += A[64 x 16] * B[N x 16]^T, kind f16 (fp32 accumulate), for the instantiated N (tc_mma_n).  rs: A from
// registers (fragment of K-step t); ss: A from a shared-memory descriptor.  Both use accumulator registers d[0, N/2):
// element e of the fragment covers columns 8(e >> 2) .. +7 whatever N is, so the columns >= N keep their value.
// R0..R5 / S0..S2: asm operand numbers of the inputs (after the N/2 accumulator operands).
template <int N> struct Wgmma;
#define DSPGN_WGMMA(N, DREGS, OPS, R0, R1, R2, R3, R4, R5, S0, S1, S2)                                          \
  template <> struct Wgmma<N> {                                                                                 \
    static __device__ __forceinline__ void rs(float (&d)[128], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, \
                                              uint64_t b_desc) {                                                \
      asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %" #R5 ", 0;\n\t"                                       \
                   "wgmma.mma_async.sync.aligned.m64n" #N "k16.f32.f16.f16 " OPS                                 \
                   "{%" #R0 ", %" #R1 ", %" #R2 ", %" #R3 "}, %" #R4 ", p, 1, 1, 0;\n\t}"                         \
                   : DREGS                                                                                      \
                   : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "l"(b_desc), "r"(1)                                    \
                   : "memory");                                                                                 \
    }                                                                                                           \
    static __device__ __forceinline__ void ss(float (&d)[128], uint64_t a_desc, uint64_t b_desc) {              \
      asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %" #S2 ", 0;\n\t"                                       \
                   "wgmma.mma_async.sync.aligned.m64n" #N "k16.f32.f16.f16 " OPS                                 \
                   "%" #S0 ", %" #S1 ", p, 1, 1, 0, 0;\n\t}"                                                     \
                   : DREGS                                                                                      \
                   : "l"(a_desc), "l"(b_desc), "r"(1)                                                           \
                   : "memory");                                                                                 \
    }                                                                                                           \
  };
DSPGN_WGMMA(256, DSPGN_D128, DSPGN_ACC_OPS128, 128, 129, 130, 131, 132, 133, 128, 129, 130)
DSPGN_WGMMA(192, DSPGN_D96, DSPGN_ACC_OPS96, 96, 97, 98, 99, 100, 101, 96, 97, 98)
DSPGN_WGMMA(80, DSPGN_D40, DSPGN_ACC_OPS40, 40, 41, 42, 43, 44, 45, 40, 41, 42)
#undef DSPGN_WGMMA

__device__ __forceinline__ void epi_bar_sync() { asm volatile("bar.sync 1, 256;" ::: "memory"); }

// ---- cycle accounting of the tile (probe build only: -DDSPGN_STALL_PROBE, tools/tile_probe.py) ----------------------
// Lane 0 of consumer warp 0 of each warpgroup and the producer lane add the clock64 cycles they spend in each part of
// the tile loop to per-CTA counters: row 0 / 1 = consumer warpgroup 0 / 1, row 2 = producer.  The shipped library
// compiles none of it.  The epilogue (PR_EPI) is split further: the barrier that opens it (PR_EPI_ENTRY), then per step
// kind (EpiKind) three slots from PR_EPI_KIND + 3 * kind: the value loop, the split and stores of store_operand, and its
// proxy fence + warpgroup barrier.  The prologue (PR_PROLOGUE) is split into its global reads with the two barriers
// (PR_PRO_GLOBAL) and the layer-0 loop with its store_operand (PR_PRO_L0); the tile's final step (PR_JTJ) into the pose
// columns and residual with their two barriers (PR_JTJ_POSE), the J^T J chains (PR_JTJ_LOOP) and the partial stores
// (PR_JTJ_STORE).  The probed lanes run J^T J, not J^T r: a J^T r that outlasts J^T J shows up in PR_TILE_END's barrier.
enum ProbeSlot {
  PR_WFULL, PR_WGWAIT, PR_GEMM, PR_EPI, PR_PROLOGUE, PR_JTJ, PR_TILE_END, PR_SOLVE, PR_FIFO, PR_LOOP, PR_TILES, PR_SOLVES,
  PR_WEMPTY, PR_POP, PR_PROD_LOOP, PR_EPI_ENTRY, PR_EPI_KIND, PR_PRO_GLOBAL = PR_EPI_KIND + 3 * 6, PR_PRO_L0, PR_JTJ_POSE,
  PR_JTJ_LOOP, PR_JTJ_STORE, kProbeSlots
};
// hidden forward, the same before latent_in (concat), last hidden layer, backward, the same at latent_in (skip gradient),
// first layer backward
enum EpiKind { EK_FWD, EK_FWD_CAT, EK_PENULT, EK_BWD, EK_BWD_SKIP, EK_BWD_FIRST };
constexpr int kProbeCtas = 256;
#ifdef DSPGN_STALL_PROBE
__device__ unsigned long long g_stall_probe[kProbeCtas * 3 * kProbeSlots];
__device__ __forceinline__ void probe_add(int slot, unsigned long long v) {
  if ((threadIdx.x & 127) == 0 && blockIdx.x < kProbeCtas)
    atomicAdd(&g_stall_probe[(blockIdx.x * 3 + (threadIdx.x >> 7)) * kProbeSlots + slot], v);
}
#define DSPGN_PROBE_T(t0) const long long t0 = clock64()
#define DSPGN_PROBE_ADD(slot, t0) probe_add(slot, (unsigned long long)(clock64() - (t0)))
#define DSPGN_PROBE_COUNT(slot) probe_add(slot, 1ull)
#define DSPGN_PROBE_ADD_IF(cond, slot, t0) do { if (cond) DSPGN_PROBE_ADD(slot, t0); } while (0)
#else
#define DSPGN_PROBE_T(t0)
#define DSPGN_PROBE_ADD(slot, t0)
#define DSPGN_PROBE_COUNT(slot)
#define DSPGN_PROBE_ADD_IF(cond, slot, t0)
#endif

// K-major, 128B-swizzled shared-memory matrix descriptor (sm90 GMMA descriptor):
// start>>4 [0,14) | LBO>>4 [16,30) = 1 (unused for swizzled K-major) | SBO>>4 [32,46) = 64 (8 rows x 128 B) |
// base offset [49,52) = 0 (1024 B aligned atoms) | layout [62,64) = 1 (SWIZZLE_128B)
__device__ __forceinline__ uint64_t make_desc(uint32_t smem_addr) {
  uint64_t d = 0;
  d |= (uint64_t)((smem_addr >> 4) & 0x3FFF);
  d |= (uint64_t)1 << 16;
  d |= (uint64_t)64 << 32;
  d |= (uint64_t)1 << 62;
  return d;
}
// same for a weight ring stage: K-major rows of 64 B (32 K), 64B-swizzled: SBO>>4 = 32 (8 rows x 64 B), layout 2
// (SWIZZLE_64B); 512 B aligned atoms
__device__ __forceinline__ uint64_t make_desc_w(uint32_t smem_addr) {
  uint64_t d = 0;
  d |= (uint64_t)((smem_addr >> 4) & 0x3FFF);
  d |= (uint64_t)1 << 16;
  d |= (uint64_t)32 << 32;
  d |= (uint64_t)2 << 62;
  return d;
}

// fp32 -> (fp16 hi, fp16 lo) for two consecutive K elements, packed low half = even element
__device__ __forceinline__ void split_pack(float a, float b, uint32_t& hi, uint32_t& lo) {
  __half2 h = __floats2half2_rn(a, b);
  float2 back = __half22float2(h);
  __half2 l = __floats2half2_rn(a - back.x, b - back.y);
  hi = *reinterpret_cast<uint32_t*>(&h);
  lo = *reinterpret_cast<uint32_t*>(&l);
}

// ------------------------------------------------------------------------------------------------
// shared-memory carve-up
// ------------------------------------------------------------------------------------------------
constexpr int kJpStride = 76;             // floats per row of the point-major Jacobian tile (72 + pad, 16B aligned)
constexpr int kTcMaskLayers = 8;          // hidden layers with a saved ReLU mask (layers 0 .. 7 of the 8 x 256 decoders)
// Shared-memory state of the persistent schedule (the mega_* helpers), embedded in the tail of every persistent kernel:
// the CTA-local tile FIFO (scheduler lane -> epilogue threads), the stage-end flag word, the copies of the kernel
// arguments for the out-of-line solve step and the cooperative publication of an object's next-iteration tiles.
// Passing references to the kernel parameters themselves would make them address-taken: the compiler then parks all of
// them in local memory and the tile loop reads its pointers with LDL instead of from the constant bank.
struct MegaSmem {
  int fifo[4]; int fifo_pub; int epi_seq; int last_flag;
  BatchDev ctx_b; MegaArgs ctx_q; SolveArgs ctx_sv;
  int push_base, push_nF, push_nS, push_o;
  // one thread, before the kernel's first barrier
  __device__ void init(const BatchDev& b, const MegaArgs& q, const SolveArgs& sv) {
    fifo_pub = 0; epi_seq = 0; last_flag = 0;
    ctx_b = b; ctx_q = q; ctx_sv = sv;
  }
};
template <int SCHED>
struct TcSmemTail {
  float Jp[kTcRows * kJpStride];          // [row][72+4]: J row of each point; cols 0..66 double as latent_in skip gradient
  // ReLU masks [layer][word][consumer thread]: bit e of word w = fragment element 32w+e.  SCHED 1 keeps them in a per-CTA
  // global scratch ([layer][consumer thread] of uint4) and stages here only the layer a backward step reads: [thread] of uint4.
  uint32_t maskw[(SCHED == 1 ? 1 : kTcMaskLayers) * 4 * kTcEpiThreads];
  float bias[9 * kHid];
  float wlast[kHid];
  float w0x[3 * kHid];                    // xyz rows of the layer-0 matrix (the latent rows are folded into ObjState.zb0)
  TileObj obj;                            // the tile's object (stage_obj)
  float xr[3 * kTcRows];                  // object-frame point of every row
  float rr[kTcRows], rsc[kTcRows];
  float yrow[kTcRows], scr[kTcRows];      // decoder output and row weight (0 = inactive row) of every row
  int prefix[SCHED == 1 ? 1 : kMaxObjScan + 1];     // tile prefix of the per-iteration schedule (unused by SCHED 1)
  int warp_tmp[32];
  uint64_t w_full[kTcRing<SCHED>], w_empty[kTcRing<SCHED>];   // adjacent: wg_gemm addresses both from w_full
  TcPlan plans[DSPGN_MAX_CLASSES];        // step plans of every decoder class (read by all warp roles)
  int cur_class;
  MegaSmem mega;                          // persistent mode (scheduler = producer warp)
  // workspace of the solve step (mega_solve_and_advance): the J tile, dead between tiles
  __device__ SolveSmem& solve_smem() { return *reinterpret_cast<SolveSmem*>(Jp); }
};
template <int SCHED>
constexpr size_t kTcSmemBytes = 1024 + (size_t)kTcRing<SCHED> * kTcStageBytes + 2 * (size_t)kTcAloBytes + sizeof(TcSmemTail<SCHED>);
static_assert(kTcSmemBytes<0> <= 227 * 1024, "k_decoder_tc: shared memory exceeds the 227 KB per block of sm_90");
static_assert(kTcSmemBytes<1> <= 227 * 1024, "k_gn_persistent: shared memory exceeds the 227 KB per block of sm_90");
static_assert(kTcSmemBytes<2> <= 227 * 1024, "k_gn_persistent_render: shared memory exceeds the 227 KB per block of sm_90");
static_assert(offsetof(TcSmemTail<0>, bias) % 8 == 0 && offsetof(TcSmemTail<0>, w0x) % 8 == 0 &&
              offsetof(TcSmemTail<1>, bias) % 8 == 0 && offsetof(TcSmemTail<1>, w0x) % 8 == 0 &&
              offsetof(TcSmemTail<2>, bias) % 8 == 0 && offsetof(TcSmemTail<2>, w0x) % 8 == 0,
              "the epilogues read bias and W0 column pairs as float2");
static_assert(offsetof(TcSmemTail<1>, maskw) % 16 == 0, "the SDF-tile kernel stages one uint4 of masks per thread");

// ---- J^T J, J^T (rho r) and the loss of a J tile of ROWS rows (optimizer.py:161-167) into its partial sums accp.  Row p
// of the tile: its Jacobian row at Jp[p * kJpStride] with rho r in column 71, rho r in rr[p], its row count in rsc[p].
// Threads 0..170: one upper-triangular 4 x 4 block of the 72 x 72 product each; column 71 is left out of H, and the
// chains of column block 17 give J^T (rho r) as  fmaf(J[p][c], rho r[p], .)  over p in order.  Threads 248..255: loss
// and row count over ROWS / 8 rows each, fixed-order combine.
template <int ROWS>
__device__ __forceinline__ void jtile_sums(const float* Jp, const float* rr, const float* rsc, float* accp, int tid) {
  if (tid < 171) {
    DSPGN_PROBE_T(tjl);
    int bi = 0, rem = tid;
    while (rem >= 18 - bi) { rem -= 18 - bi; ++bi; }
    const int bj = bi + rem;
    float h[4][4];
#pragma unroll
    for (int u = 0; u < 4; ++u)
#pragma unroll
      for (int v = 0; v < 4; ++v) h[u][v] = 0.f;
    const float* pa = Jp + 4 * bi;
    const float* pb = Jp + 4 * bj;
#pragma unroll 4
    for (int p = 0; p < ROWS; ++p) {
      const float4 A4 = *reinterpret_cast<const float4*>(pa + p * kJpStride);
      const float4 B4 = *reinterpret_cast<const float4*>(pb + p * kJpStride);
      const float av[4] = {A4.x, A4.y, A4.z, A4.w}, bv[4] = {B4.x, B4.y, B4.z, B4.w};
#pragma unroll
      for (int u = 0; u < 4; ++u)
#pragma unroll
        for (int v = 0; v < 4; ++v) h[u][v] = fmaf(av[u], bv[v], h[u][v]);
    }
    DSPGN_PROBE_ADD(PR_JTJ_LOOP, tjl);
    DSPGN_PROBE_T(tjs);
#pragma unroll
    for (int u = 0; u < 4; ++u)
#pragma unroll
      for (int v = 0; v < 4; ++v) {
        const int rI = 4 * bi + u, cI = 4 * bj + v;
        if (cI >= rI && cI < kMaxCode + 7) accp[tri_index(rI, cI)] = h[u][v];
      }
    if (bj == 17) {
#pragma unroll
      for (int u = 0; u < 4; ++u)
        if (4 * bi + u < kMaxCode + 7) accp[kAccB + 4 * bi + u] = h[u][3];
    }
    DSPGN_PROBE_ADD(PR_JTJ_STORE, tjs);
  } else if (tid >= 248) {
    constexpr int kPer = ROWS / 8;
    const int k = tid - 248;
    float sacc = 0.f, n = 0.f;
    for (int p = kPer * k; p < kPer * k + kPer; ++p) { sacc = fmaf(rr[p], rr[p], sacc); n += rsc[p]; }
#pragma unroll
    for (int d = 1; d < 8; d <<= 1) {
      sacc += __shfl_down_sync(0xff000000u, sacc, d);
      n += __shfl_down_sync(0xff000000u, n, d);
    }
    if (k == 0) { accp[kAccLoss] = sacc; accp[kAccLoss + 1] = n; }
  }
}

// ---- accumulator fragment (m64nNk16, fp32): thread (warp w of the warpgroup, lane l) holds element e of
// 8-column block j = e >> 2 at row 16w + l/4 (+8 when e & 2), column 8j + 2(l%4) + (e & 1).
__device__ __forceinline__ int frag_col(int e, int q) { return 8 * (e >> 2) + 2 * q + (e & 1); }
// The epilogues take the fragment column pair q through an opaque move made inside the tile loop.  With the plain value
// the compiler hoists the 64 distinct frag_col() results out of the loop, and they end up in local memory.
__device__ __forceinline__ int opaque_int(int v) {
  int r;
  asm volatile("mov.b32 %0, %1;" : "=r"(r) : "r"(v));
  return r;
}

// accumulator-shaped values -> A operand of the next GEMM step: hi halves into `ah` (the register A fragment of
// K-step t is columns [16t, 16t+16) of the accumulator fragment), lo halves into this warpgroup's swizzled image `alo`
// (shared-space address: 4 K chunks of 64 rows x 128 B, 128B swizzle), written with 16 stmatrix.x4.  The lo halves of
// K-step t form an m16k16 fragment whose four 8 x 8 matrices, (rows rl / rl + 8) x (columns 16t.. / 16t+8..), are
// exactly the thread's values h = 0..3, v[8t + 2h], v[8t + 2h + 1]; lane l gives the swizzled address of row l % 8 of
// matrix l / 8.  Column kk of row `row` sits at byte  (kk >> 6) * 8192 + row * 128 + ((((kk & 63) >> 3) ^ (row & 7)) << 4)
// + (kk & 7) * 2; in that 16-byte chunk the K-step enters only as 2(t & 3), so a lane needs one base address and one
// xor per t.  Ends with the proxy fence and the warpgroup barrier the wgmma reads need.  pslot: probe build only, the
// step kind's first probe slot (PR_EPI_KIND + 3 * kind), or -1.
__device__ __forceinline__ void store_operand(const float (&v)[128], uint32_t (&ah)[64], uint32_t alo, int grp, int pslot = -1) {
  DSPGN_PROBE_T(ts);
  const int lane = threadIdx.x & 31;
  const int srow = 16 * ((threadIdx.x >> 5) & 3) + (lane & 7) + 8 * ((lane >> 3) & 1);
  const uint32_t base = alo + 128u * (uint32_t)srow;
  const uint32_t xo = (uint32_t)(((lane >> 4) & 1) ^ (lane & 7)) << 4;
#pragma unroll
  for (int t = 0; t < 16; ++t) {
    uint32_t lo[4];
#pragma unroll
    for (int h = 0; h < 4; ++h) split_pack(v[8 * t + 2 * h], v[8 * t + 2 * h + 1], ah[4 * t + h], lo[h]);
    const uint32_t addr = base + 8192u * (uint32_t)(t >> 2) + (xo ^ (32u * (uint32_t)(t & 3)));
    asm volatile("stmatrix.sync.aligned.m8n8.x4.shared.b16 [%0], {%1, %2, %3, %4};" ::"r"(addr), "r"(lo[0]), "r"(lo[1]),
                 "r"(lo[2]), "r"(lo[3]) : "memory");
  }
  DSPGN_PROBE_ADD_IF(pslot >= 0, pslot + 1, ts);
  DSPGN_PROBE_T(tf);
  fence_proxy_async();
  wg_bar_sync(grp);
  DSPGN_PROBE_ADD_IF(pslot >= 0, pslot + 2, tf);
}

// ---- epilogue value loops of the tile, without a branch per fragment element.  Fragment element e = 4j + h covers
// columns 8j + 2q + (h & 1) with q < 4, and n_mma and k_next are multiples of 8: a column is below either bound iff 8j
// is.  NM / KNEXT are the step's n_mma / k_next at compile time, so for the pairs the 8 x 256 decoders produce every live
// / zero decision is fixed per j.  NM = KNEXT = 0 is the fallback for other pairs: the runtime values nm / k_next.
// Steps with more to do than bias + ReLU or the mask run it as a separate pass over the fragment: folded into one loop,
// the extra loads, stores and dot-product chain are scheduled across the whole fragment and the tile loop spills.
template <int NM, int KNEXT>
__device__ __forceinline__ void epi_fwd_hidden(float (&acc)[128], uint32_t (&mw)[4], const float* bb, int qs, int nm, int k_next) {
#pragma unroll
  for (int j = 0; j < 32; ++j) {
    const bool live = 8 * j < (NM ? NM : nm), nxt = 8 * j < (KNEXT ? KNEXT : k_next);
    const float2 bj = *reinterpret_cast<const float2*>(bb + 8 * j + 2 * qs);
#pragma unroll
    for (int h = 0; h < 4; ++h) {
      const int e = 4 * j + h;
      const float w = acc[e] + ((h & 1) ? bj.y : bj.x);
      mw[e >> 5] |= ((live && w > 0.f) ? 1u : 0u) << (e & 31);
      acc[e] = (live && nxt) ? fmaxf(w, 0.f) : 0.f;
    }
  }
}

// the layer before latent_in, after epi_fwd_hidden: columns >= cat_off below k_next take the decoder input
// [z | x | 0...] (deep_sdf_decoder.py:87-88), read from clamped shared-memory indices and selected.  Column blocks
// below cat_off are skipped whole (a branch per block, not per element).  CAT / LL: cat_off and L at compile time (189
// and 64 for the 8 x 256 decoders with a 64-wide code): the blocks that lie wholly inside the code then read it at a
// fixed offset from one lane address, and only the blocks that straddle cat_off or L select per element.  CAT = 0: the
// runtime cat_off_ / L_.
template <int CAT, int LL>
__device__ __forceinline__ void epi_concat_input(float (&acc)[128], int qs, int k_next, int cat_off_, int L_, const float* zs,
                                                 const float* xr, int rowA, int rowB) {
  const int cat_off = CAT ? CAT : cat_off_, L = CAT ? LL : L_;
#pragma unroll
  for (int j = 0; j < 32; ++j) {
    if (8 * j + 8 <= cat_off) continue;
    const bool nxt = 8 * j < k_next;
    if (CAT && 8 * j >= cat_off && 8 * j + 8 - cat_off <= L) {
#pragma unroll
      for (int h = 0; h < 4; ++h) acc[4 * j + h] = nxt ? zs[2 * qs + (8 * j + (h & 1) - cat_off)] : acc[4 * j + h];
      continue;
    }
#pragma unroll
    for (int h = 0; h < 4; ++h) {
      const int e = 4 * j + h, i = 8 * j + 2 * qs + (h & 1) - cat_off, ix = i - L;
      const float zv = zs[(unsigned)i < (unsigned)L ? i : 0];
      const float xv = xr[((unsigned)ix < 3u ? ix : 0) * kTcRows + ((h & 2) ? rowB : rowA)];
      acc[e] = (nxt && i >= 0) ? (i < L ? zv : ((unsigned)ix < 3u ? xv : 0.f)) : acc[e];
    }
  }
}

// the layer at latent_in, before epi_bwd_mid: the gradient of its skip columns (>= cat_off) goes to the Jacobian tile
// (the first in0 of them, predicated stores) instead of to the next layer.  Column blocks below cat_off are skipped
// whole.  CAT / LL as in epi_concat_input (in0 = LL + 3, and nm = 256: every column is live): the blocks wholly inside
// the code store unpredicated at a fixed offset from one lane address.
template <int CAT, int LL>
__device__ __forceinline__ void epi_skip_grad(float (&acc)[128], int qs, int nm, int cat_off_, int in0_, int L_, float* Jp, int rowA,
                                              int rowB) {
  const int cat_off = CAT ? CAT : cat_off_, L = CAT ? LL : L_, in0 = CAT ? LL + 3 : in0_;
#pragma unroll
  for (int j = 0; j < 32; ++j) {
    if (8 * j + 8 <= cat_off) continue;
    const bool live = 8 * j < (CAT ? kHid : nm);
    if (CAT && 8 * j >= cat_off && 8 * j + 8 - cat_off <= L) {
      float* pa = Jp + rowA * kJpStride + 2 * qs;
      float* pb = Jp + rowB * kJpStride + 2 * qs;
#pragma unroll
      for (int h = 0; h < 4; ++h) {
        const int e = 4 * j + h, off = 8 * j + (h & 1) - cat_off;
        ((h & 2) ? pb : pa)[off] = acc[e];
        acc[e] = 0.f;
      }
      continue;
    }
#pragma unroll
    for (int h = 0; h < 4; ++h) {
      const int e = 4 * j + h, ii = 8 * j + 2 * qs + (h & 1) - cat_off;
      if (live && ii >= 0 && ii < in0) Jp[((h & 2) ? rowB : rowA) * kJpStride + ((ii < L) ? ii : (kMaxCode + ii - L))] = acc[e];
      acc[e] = (ii >= 0) ? 0.f : acc[e];
    }
  }
}

// backward through a hidden layer: the saved ReLU mask
template <int NM, int KNEXT>
__device__ __forceinline__ void epi_bwd_mid(float (&acc)[128], const uint32_t (&mw)[4], int nm, int k_next) {
#pragma unroll
  for (int j = 0; j < 32; ++j) {
    const bool live = 8 * j < (NM ? NM : nm), nxt = 8 * j < (KNEXT ? KNEXT : k_next);
#pragma unroll
    for (int h = 0; h < 4; ++h) {
      const int e = 4 * j + h;
      acc[e] = (live && nxt && ((mw[e >> 5] >> (e & 31)) & 1u)) ? acc[e] : 0.f;
    }
  }
}

// d/d(input) of the first layer: the Jacobian row, plus the skip gradient stored before (loss.py:34-41 / :143-150).
// The step's wgmma N is always 80: tc_pack_decoder takes decoders with in0 <= 80 only, so the 10 column blocks below 80
// are the whole fragment the step computes.
__device__ __forceinline__ void epi_bwd_first(const float (&acc)[128], int qs, int in0, int L, bool has_skip, float* Jp,
                                              const float* scr, int rowA, int rowB) {
  const float sa = scr[rowA], sb = scr[rowB];
#pragma unroll
  for (int j = 0; j < 10; ++j) {
#pragma unroll
    for (int h = 0; h < 4; ++h) {
      const int c = 8 * j + 2 * qs + (h & 1);
      const bool st = c < in0;
      float* pj = Jp + ((h & 2) ? rowB : rowA) * kJpStride + (st ? ((c < L) ? c : (kMaxCode + c - L)) : 0);
      const float g = has_skip ? acc[4 * j + h] + *pj : acc[4 * j + h];
      if (st) *pj = g * ((h & 2) ? sb : sa);                       // loss.py:145 (de_ds) / inactive rows
    }
  }
}

// layer 0 of a decoder whose first GEMM step takes all 256 of its outputs (k_steps * 16 = out_dim[0] = 256): every
// column is live, bias (zb0) and the xyz rows of W0 are read as column pairs.  The fmaf order is that of the runtime
// layer-0 loop in tc_body for other shapes:  bias -> x0 -> x1 -> x2.
__device__ __forceinline__ void epi_layer0_256(float (&acc)[128], uint32_t (&mw)[4], const float* bias, const float* w0x, int qs,
                                               float xa0, float xa1, float xa2, float xb0, float xb1, float xb2) {
#pragma unroll
  for (int j = 0; j < 32; ++j) {
    const int c = 8 * j + 2 * qs;
    const float2 bj = *reinterpret_cast<const float2*>(bias + c);
    const float2 w0 = *reinterpret_cast<const float2*>(w0x + c);
    const float2 w1 = *reinterpret_cast<const float2*>(w0x + kHid + c);
    const float2 w2 = *reinterpret_cast<const float2*>(w0x + 2 * kHid + c);
#pragma unroll
    for (int h = 0; h < 4; ++h) {
      const int e = 4 * j + h;
      const bool hb = (h & 2) != 0, hy = (h & 1) != 0;
      float w = hy ? bj.y : bj.x;
      w = fmaf(hy ? w0.y : w0.x, hb ? xb0 : xa0, w);
      w = fmaf(hy ? w1.y : w1.x, hb ? xb1 : xa1, w);
      w = fmaf(hy ? w2.y : w2.x, hb ? xb2 : xa2, w);
      mw[e >> 5] |= (w > 0.f ? 1u : 0u) << (e & 31);
      acc[e] = w > 0.f ? w : 0.f;
    }
  }
}

// every consumer warp has finished reading ring stage s (its wgmma groups have completed)
__device__ __forceinline__ void release_stage(uint32_t w_empty, int s) {
  __syncwarp();
  if ((threadIdx.x & 31) == 0) mbar_arrive(w_empty + 8u * s);
}

// Position in a ring of RING stages: the ring stage `k` stages after (stage, phase), and the parity of that lap.  Producer
// and consumers each carry (stage, phase) across steps and tiles; they visit the stages in the same order.
template <int RING>
__device__ __forceinline__ void ring_at(uint32_t stage, uint32_t phase, uint32_t k, uint32_t& slot, uint32_t& par) {
  const uint32_t g = stage + k, laps = g / RING;
  slot = g - RING * laps;
  par = phase ^ (laps & 1u);
}

// One GEMM step of a consumer warpgroup: acc = A * W^T over nch K chunks of 64, W streamed through the weight ring of
// RING stages.  The stages of a chunk arrive as hi[k 0..31], hi[k 32..63], lo[k 0..31], lo[k 32..63], so every output
// element accumulates in the order  A_hi W_hi, A_lo W_hi  per K-step, then  A_hi W_lo  per K-step,  as when the chunk was
// one image pair.  Each chunk is a fixed, unrolled MMA sequence (only the chunk count varies), one commit group per stage.
// Behind every second stage `wgmma.wait_group 1` retires all but the newest group and their stages go back to the
// producer, which refills them while the newest group runs.  Stage s of chunk c sits in ring stage (stage + 4c + s) mod
// RING; a 4-stage ring holds exactly one chunk, so there every step starts at stage 0.
// alo, ring, bars: shared-space addresses (32-bit: the MMA sequence runs with few registers to spare); bars holds the
// RING full barriers followed by the RING empty barriers.
template <int N, int RING>
__device__ __forceinline__ void wg_gemm(float (&acc)[128], const uint32_t (&ah)[64], uint32_t alo, uint32_t ring,
                                        uint32_t bars, uint32_t& stage, uint32_t& phase, int nch) {
  static_assert(RING >= kTcStages, "the ring holds at least one K chunk");
  const uint32_t w_full = bars, w_empty = bars + 8u * RING;
  const uint32_t st0 = (RING == kTcStages) ? 0u : stage;
  // Every ring stage is recomputed from the step's start position: a stage index carried from one chunk to the next
  // makes ptxas serialize the wgmma (C7515).
  auto slot_of = [&](int k) { uint32_t sl, p; ring_at<RING>(st0, phase, (uint32_t)k, sl, p); return sl; };
#pragma unroll
  for (int i = 0; i < 128; ++i) acc[i] = 0.f;
#pragma unroll
  for (int c = 0; c < 4; ++c) {
    if (c < nch) {
#pragma unroll
      for (int s = 0; s < kTcStages; ++s) {
        uint32_t slot, ph;
        ring_at<RING>(st0, phase, (uint32_t)(kTcStages * c + s), slot, ph);
        DSPGN_PROBE_T(tf);
        mbar_wait(w_full + 8u * slot, ph);
        DSPGN_PROBE_ADD(PR_WFULL, tf);
        wg_fence();
        const uint32_t bw = ring + slot * kTcStageBytes;
#pragma unroll
        for (int k = 0; k < 2; ++k) {
          const int t = 4 * c + 2 * (s & 1) + k;             // K-step of the step
          const uint64_t bd = make_desc_w(bw + 32u * k);
          Wgmma<N>::rs(acc, ah[4 * t], ah[4 * t + 1], ah[4 * t + 2], ah[4 * t + 3], bd);
          if (s < 2) Wgmma<N>::ss(acc, make_desc(alo + 8192u * c + 32u * (t & 3)), bd);
        }
        wg_commit();
        if (s == 1) {
          DSPGN_PROBE_T(tw);
          wg_wait1();
          DSPGN_PROBE_ADD(PR_WGWAIT, tw);
          release_stage(w_empty, slot_of(kTcStages * c));
          if (c > 0) release_stage(w_empty, slot_of(kTcStages * c - 1));
        } else if (s == 3) {
          DSPGN_PROBE_T(tw);
          wg_wait1();
          DSPGN_PROBE_ADD(PR_WGWAIT, tw);
          release_stage(w_empty, slot_of(kTcStages * c + 1));
          release_stage(w_empty, slot_of(kTcStages * c + 2));
        }
      }
    }
  }
  DSPGN_PROBE_T(tw);
  wg_wait0();
  DSPGN_PROBE_ADD(PR_WGWAIT, tw);
  release_stage(w_empty, slot_of(kTcStages * nch - 1));
  ring_at<RING>(st0, phase, (uint32_t)(kTcStages * nch), stage, phase);
}

// producer side of the ring: the weight images of one GEMM step, nch chunks of 4 stages of img_bytes each, into the ring
// stages (STAGE_BYTES apart) from (stage, phase) on
template <int RING, int STAGE_BYTES = kTcStageBytes>
__device__ __forceinline__ void produce_step(const unsigned char* src, int nch, uint32_t img_bytes, unsigned char* ring,
                                             uint64_t* w_full, uint64_t* w_empty, uint32_t& stage, uint32_t& phase) {
  uint32_t st = (RING == kTcStages) ? 0u : stage;             // a 4-stage ring holds exactly one chunk
  for (int c = 0; c < nch; ++c) {
    for (int s = 0; s < kTcStages; ++s) {
      uint32_t slot, ph;
      ring_at<RING>(st, phase, (uint32_t)s, slot, ph);
      DSPGN_PROBE_T(te);
      mbar_wait(&w_empty[slot], ph ^ 1);
      DSPGN_PROBE_ADD(PR_WEMPTY, te);
      mbar_expect_tx(&w_full[slot], img_bytes);
      bulk_g2s(ring + (size_t)slot * STAGE_BYTES, src + (size_t)(kTcStages * c + s) * img_bytes, img_bytes, &w_full[slot]);
    }
    ring_at<RING>(st, phase, (uint32_t)kTcStages, st, phase);
  }
  stage = st;
}

// producer side of a tile: the weight images of the first ns GEMM steps of plan (tile_steps), from the class's blob
template <int RING, int STAGE_BYTES = kTcStageBytes>
__device__ __forceinline__ void produce_tile(const unsigned char* blob, const TcPlan& plan, int ns, unsigned char* ring,
                                             uint64_t* w_full, uint64_t* w_empty, uint32_t& stage, uint32_t& phase) {
  for (int s = 0; s < ns; ++s)
    produce_step<RING, STAGE_BYTES>(blob + plan.step[s].w_off, plan.step[s].k_steps / 4, 64u * (uint32_t)plan.step[s].n_mma,
                                    ring, w_full, w_empty, stage, phase);
}

// the step plans of the batch's n_classes decoder classes into shared memory (plan_of(c): class c's plan in global
// memory); all kTcThreads threads
template <class PlanOf>
__device__ __forceinline__ void stage_plans(TcPlan* dst, int n_classes, PlanOf plan_of, int tid) {
  constexpr int kWords = (int)(sizeof(TcPlan) / 4);
  for (int i = tid; i < n_classes * kWords; i += kTcThreads)
    reinterpret_cast<int*>(&dst[i / kWords])[i % kWords] = reinterpret_cast<const int*>(&plan_of(i / kWords))[i % kWords];
}

// The tile's object into shared memory: pose and depth range (threads 0..15), latent code zero padded (threads
// 0 .. kMaxCode + 15).  On the persistent schedule the last solve (another CTA) wrote them: read cache-bypassing
// once per tile and shared.  As 12 + 3 loads in every thread they were ~130 requests per tile for the same two L2 lines
// -- and on few-object batches every SM asks for them at the same moment.
__device__ __forceinline__ void stage_obj(TileObj& d, const ObjState& st, int L, int tid) {
  if (tid < 12) d.ost[tid] = ldv(&st.T_oc[tid]);
  else if (tid < 16) d.ost[tid] = ldv(&st.dmin + (tid - 12));
  if (tid < kMaxCode + 16) d.zs[tid] = (tid < L) ? ldv(&st.z[tid]) : 0.f;
}

struct TileRef { int o, row0, slot, mode, tile; };

// pop one work item for this CTA (persistent mode); -1 = no more work anywhere
// A wait that outlives kMegaTimeoutNs (wall clock, so it also holds under compute-sanitizer / a debugger) raises the
// abort flag: every CTA drains and exits, the host reports DSPGN_E_CUDA.  No __trap: a trap would poison the CUDA
// context of the whole process (the detectors on the Tracking thread live in it too).
constexpr unsigned long long kMegaTimeoutNs = 30ull * 1000ull * 1000ull * 1000ull;
__device__ inline int mega_pop(const MegaArgs& q, int n_obj) {
  for (;;) {
    const int t = atomicAdd(&q.ctr->head, 1);
    if (t >= q.q_cap) return -1;
    unsigned long long t0 = 0;
    int item = kItemNop;
    for (unsigned spins = 0;; ++spins) {
      const int v = ldv(q.q_flag + t);
      if (v != 0) { __threadfence(); item = v - 1; break; }
      if (ldv(&q.ctr->done_objects) >= n_obj || ldv(&q.ctr->abort_flag) != 0) return -1;
      __nanosleep(256);
      if ((spins & 1023u) == 1023u) {
        const unsigned long long now = globaltimer_ns();
        if (t0 == 0) t0 = now;
        else if (now - t0 > kMegaTimeoutNs) { atomicExch(&q.ctr->abort_flag, 1); return -1; }
      }
    }
    if (item != kItemNop) return item;       // filler of a reserved slot that was not needed: take the next ticket
  }
}

// The scheduler lane of a persistent kernel: pop this CTA's next work item into slot `seq` of the CTA-local FIFO, at most
// 3 entries ahead of the epilogue warps, and publish it (-1: no more work).
__device__ __forceinline__ void mega_fifo_fill(const MegaArgs& q, int n_obj, MegaSmem& S, int seq) {
  DSPGN_PROBE_T(tp);
  volatile int* es = &S.epi_seq;
  while (seq - *es >= 3) __nanosleep(64);   // the epilogue warps always make progress (bounded tile work)
  const int item = mega_pop(q, n_obj);
  DSPGN_PROBE_ADD(PR_POP, tp);
  if (item >= 0) log_event(q.log, ev_desc(EV_POPPED, item >> kItemKindShift, (item >> kItemObjShift) & kItemObjMask, item & kItemTileMask));
  reinterpret_cast<volatile int*>(S.fifo)[seq & 3] = item;
  __threadfence_block();
  *reinterpret_cast<volatile int*>(&S.fifo_pub) = seq + 1;
}

// Work item number `seq` of this CTA as a tile of ROWS rows; false once there is none.  SCHED 0: one launch per term,
// static round-robin over the launch's tiles (S.prefix: the block's tile prefix, build_tile_prefix; the kind is a.mode).
// Persistent kernels: the CTA-local FIFO (S.mega) its scheduler lane fills (mega_fifo_fill); SCHED 1 = SDF tiles only
// (SDF-only joint runs, pose-only runs: the kind is a compile-time constant), SCHED 2 = every item kind.
template <int ROWS, int SCHED, class Tail>
__device__ __forceinline__ bool tile_at(const BatchDev& b, const TermArgs& a, Tail& S, int seq, TileRef& t) {
  if constexpr (SCHED == 0) {
    const int tile = blockIdx.x + seq * gridDim.x;
    if (tile >= S.prefix[b.n_obj]) return false;
    t.o = find_object(S.prefix, b.n_obj, tile);
    t.tile = tile - S.prefix[t.o];
    t.row0 = t.tile * ROWS;
    t.slot = tile;
    t.mode = a.mode;
    return true;
  } else {
    volatile int* pub = &S.mega.fifo_pub;
    while (*pub <= seq) __nanosleep(64);         // filled by this CTA's scheduler lane, which always terminates (mega_pop)
    const int item = reinterpret_cast<volatile int*>(S.mega.fifo)[seq & 3];
    if (item < 0) return false;
    t.o = (item >> kItemObjShift) & kItemObjMask;
    t.mode = SCHED == 1 ? MODE_SDF : (item >> kItemKindShift);
    const int j = item & kItemTileMask;
    t.tile = j;
    t.row0 = j * ROWS;
    t.slot = (t.mode == MODE_BAND) ? a.tile_base_r[t.o] + j : (t.mode == MODE_SDF ? a.tile_base[t.o] + j : 0);
    return true;
  }
}

// rows of the term a tile belongs to (persistent kernel: the tile's own kind, counters written by other CTAs)
__device__ __forceinline__ int mega_rows(const BatchDev& b, const MegaArgs& q, const ObjMeta& M, int o, int mode) {
  if (mode == MODE_SDF) return M.n_pts;
  if (mode == MODE_BAND) return ldv(b.band_m + o);
  if (q.vpre != nullptr) return ldv(q.vpre + vpre_base(M, o) + M.n_rays) >> kRangeSampleBits;   // valid-sample hulls only
  return M.n_rays * b.D;
}

// The object's range words of a ray-sample tile (valid-sample-hull words: ray_sample_row) or a band tile (segment prefix:
// band_row_sample) into dst, a shared-memory buffer the tile does not use before its first barrier; 256 threads.
// Returns the band tile's segment count (0 otherwise); `compact`: the ray-sample tile's rows enumerate the hulls.
__device__ __forceinline__ int mega_stage_ranges(const MegaArgs& q, const ObjMeta& M, int o, int mode, int* dst, int tid,
                                                 bool& compact) {
  compact = mode == MODE_RAYFWD && q.vpre != nullptr;
  const int nseg = (mode == MODE_BAND) ? (M.n_rays + kSegRays - 1) / kSegRays : 0;
  const int nw = compact ? M.n_rays + 1 : (mode == MODE_BAND ? nseg + 1 : 0);
  const int* gp = compact ? q.vpre + vpre_base(M, o) : q.seg_prefix + seg_base(M, o);
  for (int i = tid; i < nw; i += kTcEpiThreads) dst[i] = __ldcg(gp + i);
  return nseg;
}

// publish `n` queue items (kind, object, tile 0..n-1): reserve slots, fence (everything the items depend on, incl. the
// counters updated just before the call), one word per slot.  One thread.
__device__ inline void mega_push(const MegaArgs& q, int kind, int o, int n) {
  if (n <= 0) return;
  const int base = atomicAdd(&q.ctr->tail, n);
  __threadfence();
  for (int j = 0; j < n; ++j) *reinterpret_cast<volatile int*>(q.q_flag + base + j) = make_item(kind, o, j) + 1;
}

// all terms of the object's current iteration are in: solve, update, queue the next iteration (or finish).  Called by
// the 256 epilogue threads of the CTA that completed the object's last outstanding tile.  ROWS: rows per tile of the
// kernel; Tail: its shared-memory tail (mega, warp_tmp, solve_smem()).
template <int ROWS, class Tail>
__device__ __noinline__ void mega_solve_and_advance(Tail& S, int o, int tid) {
  MegaSmem& P = S.mega;
  const BatchDev& b = P.ctx_b;
  const MegaArgs& q = P.ctx_q;
  const SolveArgs& sv = P.ctx_sv;
  __threadfence();
  SolveSmem& SM = S.solve_smem();
  const int it = ldv(q.obj_iter + o);
  const bool render = q.render && b.state[o].mode == DSPGN_MODE_JOINT;     // pose-only objects: SDF tiles only
  if (tid == 0) log_event(q.log, ev_desc(EV_SOLVE_BEGIN, 0, o, it));
  const int fin = solve_object<true>(b, sv, q.log, o, tid, SM, it + 1 >= b.state[o].n_iter);
  epi_bar_sync();
  // ---- the next iteration's ray samples: only the run of samples inside the unit sphere of every ray (new pose and
  // depth range, written by the solve above).  `fin` is the same in every thread (shared-memory flags).
  int vh = -1;
  if (!fin && render && q.vpre != nullptr) {
    const ObjMeta M = b.meta[o];
    if (M.n_rays > 0) vh = valid_sample_ranges<true>(M, b.state[o], b.rays, b.D, q.vpre + vpre_base(M, o), tid, kTcEpiThreads, S.warp_tmp);
  }
  // ---- publish: finished, or the tiles of the next iteration.  All 256 threads write the queue slots (one thread
  // pushing every ray tile and its flag one by one is on the single-object critical path).
  if (tid == 0) {
    log_event(q.log, ev_desc(EV_SOLVE_END, 0, o, it));
    int base = -1;
    if (fin) {
      // a gated pose-only object: the map-consistency check on its record; rejected, it wakes its joint slot (k_init
      // left the slot initialised, its iteration-0 counters set and no item queued), kept, the slot is done unrun
      // (a slot rejected at upload never gets here: its pose-only object was rejected at upload too); once the call's
      // stop is observed a rejected slot is not woken but gets its stopped record
      const int slot = (b.link != nullptr && b.state[o].mode == DSPGN_MODE_POSE) ? b.link[o] : -1;
      bool wake = slot >= 0 && gate_record(b.results, o, b.T_init, b.t_map) == DSPGN_GATE_REJECTED;
      if (wake && b.stop.word != nullptr && stop_seen(b.stop)) {
        stopped_slot_record(b.results, b.state, b.T_init, slot);
        wake = false;
      }
      __threadfence();                       // the result record before the object counts as done
      atomicAdd(&q.ctr->done_objects, (slot >= 0 && !wake) ? 2 : 1);
      if (wake) {
        const int ntF = ldv(q.ray_left + slot), ntS = (b.meta[slot].n_pts + ROWS - 1) / ROWS;
        base = atomicAdd(&q.ctr->tail, ntF + ntS);
        P.push_nF = ntF; P.push_nS = ntS; P.push_o = slot;
      }
    } else {
      // (no fence in this branch: the tail only reserves slots; state and counters are fenced below, before any slot is published)
      const ObjMeta M = b.meta[o];
      const int ntS = (M.n_pts + ROWS - 1) / ROWS;
      const int ntF = render ? ((vh >= 0 ? vh : M.n_rays * b.D) + ROWS - 1) / ROWS : 0;
      *reinterpret_cast<volatile int*>(q.obj_iter + o) = it + 1;
      *reinterpret_cast<volatile int*>(q.pending + o) = ntS + (ntF > 0 ? 1 : 0);
      *reinterpret_cast<volatile int*>(q.ray_left + o) = ntF;
      base = atomicAdd(&q.ctr->tail, ntF + ntS);  // the long chain (rays -> scan -> band -> solve) first, then the SDF tiles
      P.push_nF = ntF; P.push_nS = ntS; P.push_o = o;
    }
    P.push_base = base;
  }
  epi_bar_sync();
  const int base = P.push_base;
  if (base >= 0) {
    const int nF = P.push_nF, n = nF + P.push_nS;
    const int po = P.push_o;                  // o, or the joint slot it woke
    __threadfence();                          // this thread's share of the ray range words (thread 0: state, counters)
    epi_bar_sync();                           // ... of every thread, before the first slot is published
    for (int j = tid; j < n; j += kTcEpiThreads)
      *reinterpret_cast<volatile int*>(q.q_flag + base + j) = ((j < nF) ? make_item(MODE_RAYFWD, po, j) : make_item(MODE_SDF, po, j - nF)) + 1;
  }
}

// Scan item of a persistent kernel: occupancy scan / rendered depth / band rows of 64 rays (loss.py:84-141), no GEMM
// steps.  The CTA that finishes the object's last chunk turns the segment counts into the band-row prefix and queues the
// band tiles (ROWS rows each); when no SDF tile is outstanding either, it runs the solve step.  256 epilogue threads.
template <int ROWS, class Tail>
__device__ __forceinline__ void mega_scan_item(Tail& S, const BatchDev& b, const MegaArgs& q, const SolveArgs& sv, const TileRef& tr,
                                               int tid) {
  const int o = tr.o;
  scan_chunk(b, sv.prm.th, q.vpre, q.seg_cnt, o, tr.tile, tid);
  __threadfence();
  epi_bar_sync();
  if (tid == 0) {
    log_event(q.log, ev_desc(EV_TILE_END, tr.mode, o, tr.tile));
    *reinterpret_cast<volatile int*>(&S.mega.last_flag) = (atomicSub(q.scan_left + o, 1) == 1) ? 1 : 0;
  }
  epi_bar_sync();
  int act = *reinterpret_cast<volatile int*>(&S.mega.last_flag);
  if (act == 1) {
    // last chunk of the object: segment prefix -> band row count -> band tiles
    __threadfence();
    scan_prefix(b, q.seg_cnt, q.seg_prefix, o, tid, S.warp_tmp);
    epi_bar_sync();
    if (tid == 0) {
      __threadfence();                         // prefix / band_m / band rows before the band tiles are published
      atomicAdd(&q.ctr->valid_rows_total, (unsigned long long)ldv(b.V_count + o));   // V of this iteration is complete (roofline accounting)
      const int m = ldv(b.band_m + o);
      const int ntB = (m + ROWS - 1) / ROWS;
      atomicAdd(&q.ctr->band_rows_total, m);
      // the render term's placeholder in `pending` becomes its ntB band tiles BEFORE they can be popped
      const int left = atomicAdd(q.pending + o, ntB - 1) + ntB - 1;
      mega_push(q, MODE_BAND, o, ntB);
      *reinterpret_cast<volatile int*>(&S.mega.last_flag) = (left == 0) ? 2 : 0;
    }
    epi_bar_sync();
    act = *reinterpret_cast<volatile int*>(&S.mega.last_flag);
  } else act = 0;
  if (act == 2) mega_solve_and_advance<ROWS>(S, o, tid);
}

// Start of work item tr on the epilogue threads of a persistent kernel (ROWS rows per tile).  Thread 0 publishes `pub`
// as the epilogue's FIFO position (S.mega.epi_seq) and logs the item.  A scan item runs here: false, no GEMM tile.
// Otherwise the object goes to S.obj (stage_obj; read after the caller's next barrier), `iter` is the object's
// iteration (the inline cut) and `rows` the rows of the tile's term.
template <int ROWS, class Tail>
__device__ __forceinline__ bool mega_item_begin(Tail& S, const BatchDev& b, const TermArgs& a, const MegaArgs& q,
                                                const SolveArgs& sv, const TileRef& tr, int pub, int tid, int& iter, int& rows) {
  if (tid == 0) {
    *reinterpret_cast<volatile int*>(&S.mega.epi_seq) = pub;
    log_event(q.log, ev_desc(EV_TILE_BEGIN, tr.mode, tr.o, tr.tile));
  }
  if (tr.mode == kKindScan) {
    mega_scan_item<ROWS>(S, b, q, sv, tr, tid);
    return false;
  }
  const ObjMeta& M = b.meta[tr.o];
  stage_obj(S.obj, b.state[tr.o], b.decs[M.class_id].L, tid);
  iter = (a.cut_iter >= 0) ? ldv(q.obj_iter + tr.o) : a.iter;
  rows = mega_rows(b, q, M, tr.o, tr.mode);
  return true;
}

// End of a GEMM tile of a persistent kernel (kind `mode`, tile `tile` of object o, meta M): its partial
// sums / sdf values go out device-wide, then the object pipeline.  Per object and iteration:  ray-sample tiles (forward
// only) -> [last one] per-ray scan + band compaction -> band tiles (fwd+bwd) ;  SDF tiles (fwd+bwd) ;  [last SDF / band
// tile] solve, pose / code update, tiles of the next iteration.  The CTA that finishes the last tile of a stage runs the
// serial step with its 256 epilogue threads while every other SM keeps working on other objects.
template <bool RENDER, int ROWS, class Tail>
__device__ __forceinline__ void mega_tile_end(Tail& S, const MegaArgs& q, const ObjMeta& M, int o, int mode, int tile, int tid) {
  DSPGN_PROBE_T(tend);
  __threadfence();                             // this tile's partial sums / sdf values are visible device-wide
  epi_bar_sync();
  if (tid == 0) {
    log_event(q.log, ev_desc(EV_TILE_END, mode, o, tile));
    int act = 0;
    if (RENDER && mode == MODE_RAYFWD) { if (atomicSub(q.ray_left + o, 1) == 1) act = 1; }
    else if (atomicSub(q.pending + o, 1) == 1) act = 2;
    *reinterpret_cast<volatile int*>(&S.mega.last_flag) = act;
  }
  epi_bar_sync();
  int act = *reinterpret_cast<volatile int*>(&S.mega.last_flag);
  if (RENDER && act == 1) {
    // every ray sample of the object has its sdf value: the per-ray scan becomes 64-ray work items of its own
    if (tid == 0) {
      const int nch = (M.n_rays + kScanChunkRays - 1) / kScanChunkRays;
      *reinterpret_cast<volatile int*>(q.scan_left + o) = nch;
      __threadfence();
      mega_push(q, kKindScan, o, nch);
    }
  }
  DSPGN_PROBE_ADD(PR_TILE_END, tend);
  if (act == 2) {
    DSPGN_PROBE_T(tsv);
    mega_solve_and_advance<ROWS>(S, o, tid);
    DSPGN_PROBE_ADD(PR_SOLVE, tsv);
    DSPGN_PROBE_COUNT(PR_SOLVES);
  }
}

// masks_g (SCHED 1 only): the per-CTA ReLU mask scratch, [grid CTA][kTcMaskLayers][consumer thread]
template <int SCHED>
__device__ __forceinline__ void tc_body(const BatchDev& b, const TermArgs& a, const MegaArgs& q, const SolveArgs& sv,
                                        uint4* __restrict__ masks_g) {
  constexpr bool MEGA = SCHED != 0;
  constexpr bool RENDER = SCHED == 2;
  constexpr int RING = kTcRing<SCHED>;
  extern __shared__ unsigned char tc_smem_raw[];
  unsigned char* ring = tc_smem_raw + ((1024u - (smem_u32(tc_smem_raw) & 1023u)) & 1023u);   // stays a shared-space pointer
  TcSmemTail<SCHED>& S = *reinterpret_cast<TcSmemTail<SCHED>*>(ring + (size_t)RING * kTcStageBytes + 2 * (size_t)kTcAloBytes);
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;

  if (!MEGA) build_tile_prefix(b, a, kTcRows, S.prefix, S.warp_tmp);
  stage_plans(S.plans, b.n_classes, [&](int c) -> const TcPlan& { return b.decs[c].tc_plan; }, tid);
  if (tid == 0) {
    for (int i = 0; i < RING; ++i) { mbar_init(&S.w_full[i], 1); mbar_init(&S.w_empty[i], 8); }
    S.cur_class = -1;
    if (MEGA) S.mega.init(b, q, sv);
    fence_barrier_init();
  }
  __syncthreads();

  if (warp >= 8) {
    // ===================== weight producer ======================================================
    // The producer warpgroup gives its registers to the consumers; only warp 8 lane 0 has work.
    setmaxnreg_dec<kTcProducerRegs>();
    if (warp == 8 && lane == 0) {
      uint32_t stage = 0, phase = 0;
      DSPGN_PROBE_T(tloop);
      for (int seq = 0;; ++seq) {
        if (MEGA) mega_fifo_fill(q, b.n_obj, S.mega, seq);
        TileRef tr;
        if (!tile_at<kTcRows, SCHED>(b, a, S, seq, tr)) break;
        const int cls = b.meta[tr.o].class_id;
        produce_tile<RING>(b.decs[cls].tc_blob, S.plans[cls], tile_steps<MEGA>(S.plans[cls], tr.mode), ring, S.w_full, S.w_empty,
                           stage, phase);
      }
      DSPGN_PROBE_ADD(PR_PROD_LOOP, tloop);
    }
  } else {
    // ===================== consumer warpgroups =================================================
    setmaxnreg_inc<kTcConsumerRegs>();
    // Warpgroup g issues the MMAs of tile rows [64g, 64g+64) and runs their epilogue on the accumulator fragment.  The
    // per-row stages (prologue, pose columns, residual) use thread = tile row r (both groups hold the same row values).
    const int grp = warp >> 2;
    const int r = tid & 127;
    const int qd = lane & 3;                                   // fragment column pair
    const int rl = 16 * (warp & 3) + (lane >> 2);              // fragment rows rl, rl + 8 of the warpgroup
    const int rowA = 64 * grp + rl, rowB = rowA + 8;           // ... as tile rows
    unsigned char* const alo = ring + (size_t)RING * kTcStageBytes + (size_t)grp * kTcAloBytes;
    const uint32_t alo_s = smem_u32(alo), ring_s = smem_u32(ring);
    uint32_t stage = 0, phase = 0;
    float acc[128];
    uint32_t ah[64];
    DSPGN_PROBE_T(tloop);
    for (int seq = 0;; ++seq) {
      TileRef tr;
      DSPGN_PROBE_T(tq);
      if (!tile_at<kTcRows, SCHED>(b, a, S, seq, tr)) break;
      DSPGN_PROBE_ADD(PR_FIFO, tq);
      DSPGN_PROBE_T(tpro);
      // ---- prologue, phase A: everything that comes from global memory, then ONE barrier ------------------------------
      int iter = a.iter, term_n = 0;
      if constexpr (MEGA) {
        if (!mega_item_begin<kTcRows>(S, b, a, q, sv, tr, seq + 1, tid, iter, term_n)) continue;
      } else {
        stage_obj(S.obj, b.state[tr.o], b.decs[b.meta[tr.o].class_id].L, tid);
        term_n = term_rows(b, a, tr.o);
      }
      const int o = tr.o, row0 = tr.row0, tile = tr.slot, mode = tr.mode;
      const ObjMeta& M = b.meta[o];
      const ObjState& ost = b.state[o];
      const DecoderDev& dec = b.decs[M.class_id];
      const TcPlan& plan = S.plans[M.class_id];
      const int L = dec.L, in0 = dec.in0, n_lin = dec.n_lin;
      const bool has_skip = dec.latent_in >= 0;
      const bool grid_mode = !MEGA && mode == MODE_GRIDFWD;
      const bool fwd_only = (mode == MODE_RAYFWD || mode == MODE_PTSFWD || grid_mode);   // (a scan item never gets here)
      const int ns = tile_steps<MEGA>(plan, mode);
      const float huber_b = term_huber(a, mode, ost.mode, (RENDER && mode == MODE_BAND) ? a.huber_b1 : a.huber_b);
      float* const part = (RENDER && mode == MODE_BAND) ? a.part_r : a.part;
      const bool pts_mode = (mode == MODE_SDF || mode == MODE_PTSFWD || grid_mode);

      // per-class constants in smem (bias, last row, xyz rows of layer 0)
      if (S.cur_class != M.class_id) {
        for (int i = tid; i < n_lin * kHid; i += kTcEpiThreads) S.bias[i] = dec.bias[i / kHid][i % kHid];
        for (int i = tid; i < kHid; i += kTcEpiThreads) S.wlast[i] = dec.w_last[i];
        const float* __restrict__ w0g = dec.Wf[0] + (size_t)L * kHid;   // rows L..L+2 of the reduction-major layer-0 matrix
        for (int i = tid; i < 3 * kHid; i += kTcEpiThreads) S.w0x[i] = w0g[i];
      }
      // layer 0 with the latent part folded into a per-object bias (ObjState.zb0, refreshed by k_init / the solve step);
      // written after the per-class reload above, read after the barriers below
      S.bias[tid] = ldv(&ost.zb0[tid]);
      // pose-only inlier cut (optimizer.py:76-78): recorded while iteration `cut_iter` runs, applied afterwards
      const uint8_t* mask_in; uint8_t* mask_out;
      cut_masks(a, ost.mode, iter, mask_in, mask_out);
      // the object's range words (<= 8193 ints) of a ray-sample or band tile in the idle J tile
      const int* segp = reinterpret_cast<const int*>(S.Jp);
      bool compact = false;
      const int nseg = RENDER ? mega_stage_ranges(q, M, o, mode, reinterpret_cast<int*>(S.Jp), tid, compact) : 0;
      // surface points do not depend on anything above: fetch them before the barrier
      const int nrows = min(kTcRows, term_n - row0);
      float p0 = 0.f, p1 = 0.f, p2 = 0.f, sc = 0.f;
      if (pts_mode && r < nrows) {
        const float* pq = grid_mode ? a.grid + 3 * (size_t)(row0 + r) : b.pts + 3 * (size_t)(M.pts_off + row0 + r);
        p0 = pq[0]; p1 = pq[1]; p2 = pq[2];
        sc = (grid_mode || mask_in == nullptr || ldv(mask_in + M.pts_off + row0 + r)) ? 1.f : 0.f;
      }
      epi_bar_sync();      // (per-iteration schedule: Jp / rr of the previous tile are not written before the barrier further down;
                           //  persistent schedule: the previous tile ended with a barrier, its J tile is dead)
      // ---- phase B: this row's point in the object frame ----------------------------------------------------------------
      float Toc[12];
#pragma unroll
      for (int i = 0; i < 12; ++i) Toc[i] = S.obj.ost[i];
      float x0 = 0.f, x1 = 0.f, x2 = 0.f, res_in = 0.f;
      if (r < nrows) {
        const int rr_ = row0 + r;
        if (grid_mode) {
          x0 = p0; x1 = p1; x2 = p2;
        } else if (pts_mode) {
          xform_point(Toc, p0, p1, p2, x0, x1, x2);
        } else if (mode == MODE_BAND) {
          // band rows were written by the CTAs that ran this object's scan: L2 is the point of coherence
          const size_t sidx = RENDER ? band_row_sample(segp, nseg, M.smp_off, (size_t)kSegRays * b.D, rr_) : (size_t)M.smp_off + rr_;
          x0 = __ldcg(b.band_x + 3 * sidx); x1 = __ldcg(b.band_x + 3 * sidx + 1); x2 = __ldcg(b.band_x + 3 * sidx + 2);
          sc = __ldcg(b.band_s + sidx); res_in = __ldcg(b.band_r + sidx);
        } else {
          sc = ray_sample_row(b, M, Toc, S.obj.ost[12], S.obj.ost[13], S.obj.ost[14], segp, compact, rr_, x0, x1, x2);
        }
      }
      if (grp == 0) { S.xr[r] = x0; S.xr[kTcRows + r] = x1; S.xr[2 * kTcRows + r] = x2; S.scr[r] = sc; }
      epi_bar_sync();                                // zs / xr / bias visible; previous tile fully drained
      DSPGN_PROBE_ADD(PR_PRO_GLOBAL, tpro);
      DSPGN_PROBE_T(tl0);
      if (tid == 0) S.cur_class = M.class_id;

      uint32_t* const maskw = S.maskw + tid;           // word w of layer l: maskw[(4 * l + w) * kTcEpiThreads]
      // SCHED 1: this thread's masks of layer l in the CTA's global scratch (16 bytes, written once per tile by the
      // forward step, read once by a backward step)
      auto mask_g = [&](int l) { return masks_g + ((size_t)blockIdx.x * kTcMaskLayers + l) * kTcEpiThreads + tid; };
      auto save_mask = [&](int l, const uint32_t (&mw)[4]) {
        if (SCHED == 1) {
          *mask_g(l) = make_uint4(mw[0], mw[1], mw[2], mw[3]);
        } else {
#pragma unroll
          for (int w = 0; w < 4; ++w) maskw[(4 * l + w) * kTcEpiThreads] = mw[w];
        }
      };
      auto put_operand = [&](int pslot) { store_operand(acc, ah, alo_s, grp, pslot); };

      // ---- A operand of the first GEMM step (= layer 1): layer 0 on the CUDA cores.  With W0[:, :L] z folded into
      // zb0, layer 0 is 3 FMAs per output:  h0[j] = relu(zb0[j] + W0[j][L..L+2] . x)  (deep_sdf_decoder.py:91,103).
      {
        const int kk = plan.step[0].k_steps * 16;
        const int n0out = dec.out_dim[0];
        const float* w0x = S.w0x;
        const float xa0 = S.xr[rowA], xa1 = S.xr[kTcRows + rowA], xa2 = S.xr[2 * kTcRows + rowA];
        const float xb0 = S.xr[rowB], xb1 = S.xr[kTcRows + rowB], xb2 = S.xr[2 * kTcRows + rowB];
        const int qs = opaque_int(qd);
        uint32_t mw[4] = {0u, 0u, 0u, 0u};
        if (kk == kHid && n0out == kHid) {
          epi_layer0_256(acc, mw, S.bias, w0x, qs, xa0, xa1, xa2, xb0, xb1, xb2);
        } else {
#pragma unroll
          for (int e = 0; e < 128; ++e) {
            const int c = frag_col(e, qs);
            const bool hb = (e & 2) != 0;
            float w = S.bias[c];
            w = fmaf(w0x[c], hb ? xb0 : xa0, w);
            w = fmaf(w0x[kHid + c], hb ? xb1 : xa1, w);
            w = fmaf(w0x[2 * kHid + c], hb ? xb2 : xa2, w);
            const bool on = (c < kk) && (c < n0out) && (w > 0.f);
            mw[e >> 5] |= (on ? 1u : 0u) << (e & 31);
            acc[e] = on ? w : 0.f;
          }
        }
        save_mask(0, mw);
        put_operand(-1);
      }
      DSPGN_PROBE_ADD(PR_PRO_L0, tl0);
      DSPGN_PROBE_ADD(PR_PROLOGUE, tpro);
      DSPGN_PROBE_COUNT(PR_TILES);

      float yv = 0.f;
      for (int s = 0; s < ns; ++s) {
        const TcStep st = plan.step[s];
        const bool more = (s + 1 < ns);
        const int k_next = more ? plan.step[s + 1].k_steps * 16 : 0;
        const int nm = st.n_mma;
        if (MEGA && tid == 0 && s == 0) log_event(q.log, ev_desc(EV_FIRST_MMA, tr.mode, tr.o, tr.tile));
        const int nch = st.k_steps / 4;
        // SCHED 1: the masks a backward step needs are copied into the staging slot while its GEMM runs.  Each thread
        // copies and later reads only its own 16 bytes, which it stored itself in the forward pass: cp.async is a weak
        // memory operation of the issuing thread, ordered after that store, so neither a fence nor a barrier is needed.
        if (SCHED == 1 && st.kind == TK_BWD_MID) cp_async_16(smem_u32(S.maskw) + 16u * (uint32_t)tid, mask_g(st.mask_layer));
        DSPGN_PROBE_T(tg);
        if (nm == 80) wg_gemm<80, RING>(acc, ah, alo_s, ring_s, smem_u32(S.w_full), stage, phase, nch);
        else if (nm == 192) wg_gemm<192, RING>(acc, ah, alo_s, ring_s, smem_u32(S.w_full), stage, phase, nch);
        else wg_gemm<256, RING>(acc, ah, alo_s, ring_s, smem_u32(S.w_full), stage, phase, nch);
        DSPGN_PROBE_ADD(PR_GEMM, tg);
        DSPGN_PROBE_T(tepi);
        wg_bar_sync(grp);                                // every MMA of the warpgroup has read the A lo image
        DSPGN_PROBE_ADD(PR_EPI_ENTRY, tepi);
        DSPGN_PROBE_T(tval);
#ifdef DSPGN_STALL_PROBE
        const int pk = PR_EPI_KIND + 3 * (st.kind == TK_FWD_PENULT ? EK_PENULT
                                          : st.kind == TK_FWD_HIDDEN ? (st.cat_off >= 0 ? EK_FWD_CAT : EK_FWD)
                                          : st.kind == TK_BWD_MID ? (st.cat_off >= 0 ? EK_BWD_SKIP : EK_BWD) : EK_BWD_FIRST);
#else
        constexpr int pk = -1;
#endif
        const int qs = opaque_int(qd);

        if (st.kind == TK_FWD_PENULT) {
          // ---- last hidden layer: bias + ReLU (mask saved), and the final Linear(width, 1) + tanh right here as a per-row
          // dot product on the CUDA cores while the values are in registers (one GEMM step with N = 1 saved).
          // deep_sdf_decoder.py:91,103,107-108.  The 4 lanes of a quad hold one row pair: combined in a fixed order.
          const float* bb = S.bias + st.layer * kHid;
          float pa = 0.f, pb = 0.f;
          uint32_t mw[4] = {0u, 0u, 0u, 0u};
#pragma unroll
          for (int e = 0; e < 128; ++e) {
            const int c = frag_col(e, qs);
            if (c < nm) {
              const float w = acc[e] + bb[c];
              mw[e >> 5] |= (w > 0.f ? 1u : 0u) << (e & 31);
              if (e & 2) pb = fmaf(fmaxf(w, 0.f), S.wlast[c], pb);
              else pa = fmaf(fmaxf(w, 0.f), S.wlast[c], pa);
            }
          }
          save_mask(st.layer, mw);
          pa += __shfl_xor_sync(0xffffffffu, pa, 1);
          pb += __shfl_xor_sync(0xffffffffu, pb, 1);
          pa += __shfl_xor_sync(0xffffffffu, pa, 2);
          pb += __shfl_xor_sync(0xffffffffu, pb, 2);
          const float blast = S.bias[(st.layer + 1) * kHid];
          const float ya = tanhf(pa + blast), yb = tanhf(pb + blast);           // deep_sdf_decoder.py:107-108
          if (qd == 0) { S.yrow[rowA] = ya; S.yrow[rowB] = yb; }
          epi_bar_sync();
          yv = S.yrow[r];
          if (fwd_only) {
            if (grp == 0 && r < nrows) {
              const size_t base = (mode == MODE_RAYFWD) ? (size_t)M.smp_off
                                  : (grid_mode ? (size_t)a.grid_slot[o] * a.grid_rows : (size_t)M.pts_off);
              b.sdf[base + row0 + r] = (sc != 0.f) ? yv : INFINITY;
            }
            if (!RENDER && mode == MODE_RAYFWD) {        // (persistent kernel: counted by the scan items, dspgn_solve.cuh)
              const unsigned bal = __ballot_sync(0xffffffffu, grp == 0 && r < nrows && sc != 0.f);
              if (lane == 0 && bal) atomicAdd(b.V_count + o, __popc(bal));
            }
          }
          if (more) {
            // seed of the backward chain: g = (1 - y^2) W_last, masked by this layer's ReLU
            const float ga = 1.f - ya * ya, gb = 1.f - yb * yb;
#pragma unroll
            for (int e = 0; e < 128; ++e) {
              const int c = frag_col(e, qs);
              acc[e] = ((mw[e >> 5] >> (e & 31)) & 1u) ? ((e & 2) ? gb : ga) * S.wlast[c] : 0.f;
            }
            DSPGN_PROBE_ADD(pk, tval);
            put_operand(pk);
          } else {
            DSPGN_PROBE_ADD(pk, tval);
          }
        } else if (st.kind == TK_FWD_HIDDEN) {
          const float* bb = S.bias + st.layer * kHid;
          uint32_t mw[4] = {0u, 0u, 0u, 0u};
          if (nm == 256 && k_next == 256) epi_fwd_hidden<256, 256>(acc, mw, bb, qs, nm, k_next);
          else if (nm == 192 && k_next == 256) epi_fwd_hidden<192, 256>(acc, mw, bb, qs, nm, k_next);
          else epi_fwd_hidden<0, 0>(acc, mw, bb, qs, nm, k_next);
          if (st.cat_off == 189 && L == 64) epi_concat_input<189, 64>(acc, qs, k_next, st.cat_off, L, S.obj.zs, S.xr, rowA, rowB);
          else if (st.cat_off >= 0) epi_concat_input<0, 0>(acc, qs, k_next, st.cat_off, L, S.obj.zs, S.xr, rowA, rowB);
          save_mask(st.layer, mw);
          DSPGN_PROBE_ADD(pk, tval);
          put_operand(pk);
        } else if (st.kind == TK_BWD_MID) {
          uint32_t mw[4];
          if (SCHED == 1) {
            cp_async_wait_all();
            const uint4 m = reinterpret_cast<const uint4*>(S.maskw)[tid];
            mw[0] = m.x; mw[1] = m.y; mw[2] = m.z; mw[3] = m.w;
          } else {
#pragma unroll
            for (int w = 0; w < 4; ++w) mw[w] = maskw[(4 * st.mask_layer + w) * kTcEpiThreads];
          }
          if (st.cat_off == 189 && L == 64 && in0 == 67 && nm == kHid) epi_skip_grad<189, 64>(acc, qs, nm, st.cat_off, in0, L, S.Jp, rowA, rowB);
          else if (st.cat_off >= 0) epi_skip_grad<0, 0>(acc, qs, nm, st.cat_off, in0, L, S.Jp, rowA, rowB);
          if (nm == 256 && k_next == 256) epi_bwd_mid<256, 256>(acc, mw, nm, k_next);
          else if (nm == 256 && k_next == 192) epi_bwd_mid<256, 192>(acc, mw, nm, k_next);
          else epi_bwd_mid<0, 0>(acc, mw, nm, k_next);
          DSPGN_PROBE_ADD(pk, tval);
          if (more) put_operand(pk);
        } else {
          // ---- TK_BWD_FIRST: d/d(input) complete -> Jacobian row (loss.py:34-41 / :143-150) -------------
          epi_bwd_first(acc, qs, in0, L, has_skip, S.Jp, S.scr, rowA, rowB);
          DSPGN_PROBE_ADD(pk, tval);
        }
        if (!more || st.kind == TK_BWD_FIRST) {
          // no next operand: overwriting the register A fragment ends its live range at the GEMM above.  Otherwise it
          // would stay live through this epilogue (for the loop's next wg_gemm) and push the epilogue into local memory.
#pragma unroll
          for (int i = 0; i < 64; ++i) ah[i] = 0u;
        }
        DSPGN_PROBE_ADD(PR_EPI, tepi);
      }
      DSPGN_PROBE_T(tjtj);
      if (!fwd_only) {
      // ---- pose columns, residual (thread = row; needs every d/d(input) column of the row) -----------
      epi_bar_sync();
      if (grp == 0) {
        float* jr = S.Jp + r * kJpStride;
        for (int i = L; i < kMaxCode; ++i) jr[i] = 0.f;
        const RowTail t = row_tail(jr, 1, x0, x1, x2, jr[kMaxCode], jr[kMaxCode + 1], jr[kMaxCode + 2],
                                   (mode == MODE_SDF) ? yv : res_in, sc, r, nrows, mode, ost.mode, huber_b, mask_out,
                                   M.pts_off + row0);
        S.rr[r] = t.rho_r;
        jr[kMaxCode + 7] = t.rho_r;                       // for jtile_sums: J^T (rho r) from the J^T J chains
        S.rsc[r] = t.n;
        if (a.dbg_J != nullptr && o == a.dbg_obj && mode == MODE_SDF && r < nrows) a.dbg_res[row0 + r] = t.res;
      }
      epi_bar_sync();
      DSPGN_PROBE_ADD(PR_JTJ_POSE, tjtj);
      if (a.dbg_J != nullptr && o == a.dbg_obj && mode == MODE_SDF)
        dbg_dump_J(a, S.Jp, kJpStride, 1, row0, nrows, ost.mode, tid, kTcEpiThreads);
      jtile_sums<kTcRows>(S.Jp, S.rr, S.rsc, part + (size_t)tile * kAccStride, tid);
      }   // !fwd_only
      DSPGN_PROBE_ADD(PR_JTJ, tjtj);
      if (MEGA) mega_tile_end<RENDER, kTcRows>(S, q, M, o, mode, tr.tile, tid);
      // the next tile's prologue starts with epi_bar_sync(): Jp / rr are not rewritten before it
    }
    DSPGN_PROBE_ADD(PR_LOOP, tloop);
  }
}

__global__ void __launch_bounds__(kTcThreads, 1) k_decoder_tc(BatchDev b, TermArgs a) {
  tc_body<0>(b, a, MegaArgs{}, SolveArgs{}, nullptr);
}
// persistent object-pipelined variants: all GN iterations of all objects in ONE launch.
// k_gn_persistent: SDF tiles only (SDF-only joint runs, pose-only runs); k_gn_persistent_render: joint runs with the
// render term (ray-sample tiles, scan items, band tiles, SDF tiles)
// masks: ReLU mask scratch of kTcMaskLayers x kTcEpiThreads uint4 per CTA of the grid (the grid is at most the SM count)
__global__ void __launch_bounds__(kTcThreads, 1) k_gn_persistent(BatchDev b, TermArgs a, MegaArgs q, SolveArgs sv, uint4* masks) {
  tc_body<1>(b, a, q, sv, masks);
}
__global__ void __launch_bounds__(kTcThreads, 1) k_gn_persistent_render(BatchDev b, TermArgs a, MegaArgs q, SolveArgs sv) {
  tc_body<2>(b, a, q, sv, nullptr);
}

// ------------------------------------------------------------------------------------------------
// self-test kernel: D[128 x n_mma] = A[128 x 16*k_steps] * B^T through exactly the same operand paths
// (register hi / swizzled shared-memory lo A operand, swizzled weight images through the ring, 3-pass split).
// Used by tests only.
// ------------------------------------------------------------------------------------------------
constexpr size_t kTcSelftestSmem = 1024 + (size_t)kTcStages * kTcStageBytes + 2 * (size_t)kTcAloBytes + 64;
__global__ void __launch_bounds__(kTcThreads, 1) k_tc_selftest(const float* __restrict__ A, int lda, const unsigned char* __restrict__ blob,
                                                               int n_mma, int k_steps, float* __restrict__ D) {
  extern __shared__ unsigned char st_raw[];
  unsigned char* ring = st_raw + ((1024u - (smem_u32(st_raw) & 1023u)) & 1023u);
  uint64_t* bars = reinterpret_cast<uint64_t*>(ring + (size_t)kTcStages * kTcStageBytes + 2 * (size_t)kTcAloBytes);
  uint64_t* w_full = bars;
  uint64_t* w_empty = bars + kTcStages;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  if (tid == 0) {
    for (int i = 0; i < kTcStages; ++i) { mbar_init(&w_full[i], 1); mbar_init(&w_empty[i], 8); }
    fence_barrier_init();
  }
  __syncthreads();
  const int n_img = tc_mma_n(n_mma), nch = tc_pad_k_steps(k_steps) / 4;
  uint32_t stage = 0, phase = 0;
  if (warp >= 8) {
    setmaxnreg_dec<kTcProducerRegs>();
    if (warp == 8 && lane == 0) produce_step<kTcStages>(blob, nch, 64u * (uint32_t)n_img, ring, w_full, w_empty, stage, phase);
    return;
  }
  setmaxnreg_inc<kTcConsumerRegs>();
  const int grp = warp >> 2, qd = lane & 3, rl = 16 * (warp & 3) + (lane >> 2);
  const int rowA = 64 * grp + rl, rowB = rowA + 8;
  unsigned char* alo = ring + (size_t)kTcStages * kTcStageBytes + (size_t)grp * kTcAloBytes;
  float acc[128];
  uint32_t ah[64];
#pragma unroll
  for (int e = 0; e < 128; ++e) {
    const int c = frag_col(e, qd);
    acc[e] = (c < k_steps * 16) ? A[(size_t)((e & 2) ? rowB : rowA) * lda + c] : 0.f;
  }
  store_operand(acc, ah, smem_u32(alo), grp);
  if (n_img == 80) wg_gemm<80, kTcStages>(acc, ah, smem_u32(alo), smem_u32(ring), smem_u32(bars), stage, phase, nch);
  else if (n_img == 192) wg_gemm<192, kTcStages>(acc, ah, smem_u32(alo), smem_u32(ring), smem_u32(bars), stage, phase, nch);
  else wg_gemm<256, kTcStages>(acc, ah, smem_u32(alo), smem_u32(ring), smem_u32(bars), stage, phase, nch);
#pragma unroll
  for (int e = 0; e < 128; ++e) {
    const int c = frag_col(e, qd);
    if (c < n_mma) D[(size_t)((e & 2) ? rowB : rowA) * n_mma + c] = acc[e];
  }
}

// ------------------------------------------------------------------------------------------------
// host side: plan + weight images
// ------------------------------------------------------------------------------------------------
struct TcDecoderHost {
  bool ok = false;
  void* blob = nullptr;
  size_t blob_bytes = 0;
};

// images of B[n][kk] (n < n_img, kk < 16 k_steps) as fp16 hi / lo for the ring (wg_gemm / produce_step): per 64-wide K
// chunk c the four stages hi[64c, 64c+32), hi[64c+32, 64c+64), lo[...), lo[...), each n_img K-major rows of 64 B with
// 64B swizzle.  n_img is the step's wgmma N (tc_mma_n), k_steps a multiple of 4 (tc_pad_k_steps); elem returns 0 for the
// padding rows and columns.
template <class F>
inline void tc_pack_images(std::vector<unsigned char>& out, int n_img, int k_steps, F&& elem) {
  const int nch = k_steps / 4;
  const size_t img = (size_t)n_img * 64;
  const size_t base = out.size();
  out.resize(base + (size_t)nch * kTcStages * img, 0);
  for (int c = 0; c < nch; ++c)
    for (int half = 0; half < 2; ++half) {
      unsigned char* hi = out.data() + base + (size_t)(kTcStages * c + half) * img;
      unsigned char* lo = hi + 2 * img;
      for (int n = 0; n < n_img; ++n)
        for (int e = 0; e < 32; ++e) {
          const float w = elem(n, c * 64 + half * 32 + e);
          const __half h = __float2half_rn(w);
          const __half l = __float2half_rn(w - __half2float(h));
          const size_t off = (size_t)n * 64 + (size_t)(((e >> 3) ^ ((n >> 1) & 3)) << 4) + (size_t)(e & 7) * 2;
          memcpy(hi + off, &h, 2);
          memcpy(lo + off, &l, 2);
        }
    }
}

inline int round16(int x) { return (x + 15) / 16 * 16; }

inline int tc_pack_decoder(const DspgnDecoderSpec& spec, const float* const* W, const float* const* b, TcDecoderHost& h,
                           DecoderDev* dv, std::string& err) {
  (void)b;
  h.ok = false;
  dv->tc_blob = nullptr;
  memset(&dv->tc_plan, 0, sizeof(TcPlan));
  const int nl = spec.num_linear, in0 = spec.latent_size + 3, li = dv->latent_in;
  if (nl != 9 && nl < 3) return 0;
  if (in0 > 80) return 0;
  for (int k = 0; k < nl; ++k)               // the widest wgmma N is 256 (tc_mma_n): wider layers stay on the SIMT engine
    if (spec.in_dim[k] > kHid || spec.out_dim[k] > kHid) return 0;
  TcPlan& P = dv->tc_plan;
  std::vector<unsigned char> blob;
  int ns = 0;
  // forward steps: layer k, A = activations (K = in_dim), B[n][kk] = W_k[n][kk].  The final Linear(width, 1) is not a
  // GEMM step: it is folded into the epilogue of the last hidden layer (TK_FWD_PENULT) as a dot product.
  // Layer 0 is no GEMM step either: with its latent part folded into a per-object bias (ObjState.zb0) it is 3 FMAs per
  // output and is evaluated while the first operand is built (tc_body prologue).
  if (nl < 4 || li == 1) return 0;          // needs a hidden GEMM layer after layer 0 and no concat at layer 1
  for (int k = 1; k < nl - 1; ++k) {
    TcStep& s = P.step[ns];
    const int nin = spec.in_dim[k], nout = spec.out_dim[k];
    s.kind = (k == nl - 2) ? TK_FWD_PENULT : TK_FWD_HIDDEN;
    s.n_mma = tc_mma_n(nout);
    s.k_steps = tc_pad_k_steps(round16(nin) / 16);
    s.a_reg = ns & 1; s.d_reg = (ns & 1) ^ 1;
    s.layer = k; s.n_real = nout;
    s.cat_off = (k + 1 == li) ? nout : -1;
    s.mask_layer = -1;
    s.w_off = (unsigned)blob.size();
    const float* Wk = W[k];
    tc_pack_images(blob, s.n_mma, s.k_steps, [&](int n, int kk) { return (n < nout && kk < nin) ? Wk[(size_t)n * nin + kk] : 0.f; });
    ++ns;
  }
  P.n_fwd = ns;
  // backward steps: layer k = nl-2 .. 0, A = masked gradient (K = out_dim), B[n][kk] = W_k[kk][n]
  int a_reg = P.step[ns - 1].a_reg;          // the seed overwrites the (dead) A operand of the last forward GEMM step
  for (int k = nl - 2; k >= 0; --k) {
    TcStep& s = P.step[ns];
    const int nin = spec.in_dim[k], nout = spec.out_dim[k];
    s.kind = (k == 0) ? TK_BWD_FIRST : TK_BWD_MID;
    s.n_mma = tc_mma_n(nin);
    s.k_steps = tc_pad_k_steps(round16(nout) / 16);
    s.a_reg = a_reg; s.d_reg = a_reg ^ 1;
    a_reg ^= 1;
    s.layer = k; s.n_real = nin;
    s.cat_off = (k == li) ? nin - in0 : -1;
    s.mask_layer = (k > 0) ? k - 1 : -1;
    s.w_off = (unsigned)blob.size();
    const float* Wk = W[k];
    tc_pack_images(blob, s.n_mma, s.k_steps, [&](int n, int kk) { return (n < nin && kk < nout) ? Wk[(size_t)kk * nin + n] : 0.f; });
    ++ns;
  }
  P.n_steps = ns;
  // the operand of step s+1 must have been produced for k_steps(s+1)*16 columns by step s
  void* d = nullptr;
  if (cudaMalloc(&d, blob.size()) != cudaSuccess) { cudaGetLastError(); err = "cudaMalloc(tc blob)"; return DSPGN_E_ALLOC; }
  if (cudaMemcpy(d, blob.data(), blob.size(), cudaMemcpyHostToDevice) != cudaSuccess) { cudaFree(d); err = "cudaMemcpy(tc blob)"; return DSPGN_E_CUDA; }
  h.blob = d; h.blob_bytes = blob.size(); h.ok = true;
  dv->tc_blob = reinterpret_cast<const unsigned char*>(d);
  return 0;
}

inline void tc_free_decoder(TcDecoderHost& h) {
  if (h.blob) cudaFree(h.blob);
  h.blob = nullptr; h.ok = false;
}

inline int tc_setup_kernels(std::string& err) {
  if (cudaFuncSetAttribute(k_decoder_tc, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kTcSmemBytes<0>) != cudaSuccess) {
    err = std::string("cudaFuncSetAttribute(k_decoder_tc): ") + cudaGetErrorString(cudaGetLastError());
    return DSPGN_E_CUDA;
  }
  if (cudaFuncSetAttribute(k_gn_persistent, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kTcSmemBytes<1>) != cudaSuccess ||
      cudaFuncSetAttribute(k_gn_persistent_render, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kTcSmemBytes<2>) != cudaSuccess) {
    err = std::string("cudaFuncSetAttribute(k_gn_persistent): ") + cudaGetErrorString(cudaGetLastError());
    return DSPGN_E_CUDA;
  }
  if (cudaFuncSetAttribute(k_tc_selftest, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kTcSelftestSmem) != cudaSuccess) {
    err = std::string("cudaFuncSetAttribute(k_tc_selftest): ") + cudaGetErrorString(cudaGetLastError());
    return DSPGN_E_CUDA;
  }
  return 0;
}

inline bool tc_engine_default() { return true; }

inline int tc_launch_term(const BatchDev& b, const TermArgs& a, int num_sms, long long tiles_upper, cudaStream_t stream,
                          std::string& err) {
  int grid = (int)std::min<long long>(tiles_upper, num_sms);
  if (grid < 1) grid = 1;
  k_decoder_tc<<<grid, kTcThreads, kTcSmemBytes<0>, stream>>>(b, a);
  (void)err;
  return 0;
}

}  // namespace dspgn
