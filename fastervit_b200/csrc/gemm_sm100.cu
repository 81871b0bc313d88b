// fvit_gemm: persistent, warp-specialised wgmma GEMM for sm_90a.
//
//   warp 12     : TMA producer (one lane; warps 13..15 of its warpgroup only give their registers to the
//                 epilogue) — cp.async.bulk.tensor boxes into a ring of 128B-swizzled shared-memory stages,
//                 mbarrier complete_tx signalling; it runs ahead into the next tiles
//   warps 0..7  : two MMA warpgroups — wgmma.mma_async m64 x N x 16, warpgroup g owns rows [64g, 64g + 64)
//                 of the 128-row tile with fp32 accumulators in registers. N is the tile's width rounded up
//                 to 16, per work unit: a partial last N tile issues only the columns it has. At the end of
//                 a unit both wait for acc_empty, write the accumulators to the shared-memory accumulator
//                 tile, arrive on acc_full and start the next unit's K loop at once
//   warps 8..11 : the epilogue warpgroup — waits for acc_full, runs the epilogue from the accumulator tile
//                 (fused scale/shift/activation/layer-scale/residual, optional per-column statistics,
//                 row-map scatter, coalesced 16-byte global accesses) and arrives on acc_empty after its
//                 last read of the tile, so one unit's epilogue overlaps the next unit's MMAs
//
// The A operand of K-block kb is the 2-D box at row (m0 + tap_shift[tap]) of plane tap_plane[tap]:
// with 9 taps this is an im2col-free 3x3 convolution over a zero-bordered NHWC activation matrix
// (out-of-range rows are zero-filled by TMA). See include/fvit.h for the exact contract.
//
// Slab mode (stride-1 3x3 taps, tap_shift[3 dy + dx] = (dy - 1) P + (dx - 1) on one plane, kc > 128): the three
// taps of a kernel row read the same activation rows one row apart, so per (K block, dy) the producer loads one
// 136-row slab, rows
// m0 + (dy - 1) P - 1 .. +136, into a two-buffer slab ring, and only the weight tiles go through the stage ring (one
// stage per tap and K block). Tap dx of MMA warpgroup g reads slab rows [64g + dx, 64g + dx + 64). The K loop runs
// in (K block, dy, dx) order. Per K block this moves 3 x 17 KB of A instead of 9 x 16 KB.
#include <cuda_fp16.h>
#include <cuda_bf16.h>

#include <mutex>
#include <map>
#include <tuple>

#include "../../include/fvit.h"
#include "common.h"
#include "ptx.cuh"

namespace fvit {

constexpr int BM = 128;
constexpr int BK = 64;  // 64 x 16-bit = 128 B: one SWIZZLE_128B row
constexpr int MMA_K = 16;
constexpr int MMA_WARPS = 8;                    // two MMA warpgroups, each owning 64 rows of the tile
constexpr int MMA_THREADS = 32 * MMA_WARPS;
constexpr int NEPI = 4;                         // epilogue warps: one warpgroup
constexpr int EPI_THREADS = 32 * NEPI;
constexpr int TMA_WARP = MMA_WARPS + NEPI;      // first warp of the producer warpgroup (its other 3 warps idle)
constexpr int GEMM_THREADS = MMA_THREADS + EPI_THREADS + 128;
// Registers per thread (launch: 128). Every SM sub-partition holds one warp of each warpgroup, so the producer's
// surplus goes to the epilogue: 40 + 128 + 128 + 216 = 4 x 128.
constexpr uint32_t PRODUCER_REGS = 40;
constexpr uint32_t EPILOGUE_REGS = 216;
constexpr int MAX_STAGES = 12;
constexpr int A_STAGE_BYTES = BM * BK * 2;  // 16 KB
constexpr int SLAB_ROWS = BM + 8;           // slab mode: the 128 + 2 rows of three dx taps, rounded up to 8 rows
constexpr int SLAB_BYTES = SLAB_ROWS * BK * 2;  // 17 KB: a whole number of 1024-byte swizzle patterns
constexpr int SLAB_BUFS = 2;
constexpr int MAX_TILE_N = 128;             // widest MMA of the kernel (the accumulator tile lives in shared memory)
constexpr int SMEM_BUDGET = 227 * 1024;
constexpr int SMEM_CTRL_BYTES = 1024;  // barriers, placed after the stage ring
constexpr int SMEM_ALIGN_SLACK = 1024;
constexpr int ACC_LD = MAX_TILE_N + 4;  // floats per accumulator row: conflict-free float4 rows (4 banks apart)
constexpr int SMEM_ACC_BYTES = BM * ACC_LD * 4;
constexpr int STATS_MAX_N = 1024;                    // widest GEMM with per-column statistics (BatchNorm channels)
constexpr int SMEM_STATS_BYTES = 2 * STATS_MAX_N * 4;

struct GemmParams {
  int m, n;
  int num_kb;      // K-blocks (of 64) over all taps
  int kb_per_tap;  // ceil(kc / 64)
  int k_tail16;    // 16-wide MMA steps that hold real K columns in a tap's last K-block (1..4); the rest is zero fill
  int a_mn, b_mn;
  int a_row_off, b_row_off;
  int tile_n;
  int tiles_m, tiles_n, split_k;
  int b_ntaps, tiles_per_tap;  // >1: N tiles enumerate (tap, n tile); tap t reads B rows shifted by tap_shift[t]
  int atomic_out;  // split-K style accumulation: atomicAdd(alpha * acc) into out_f32
  int stages;
  int slab_pitch;  // > 0: slab mode (see the top of this file); the row pitch P of the 3x3 taps
  int tap_shift[16];
  int tap_plane[16];
  // epilogue
  float alpha;
  int act;
  int bf16;
  int vec_ok;
  const float* col_scale;
  const float* col_shift;
  const float* col_scale2;
  const void* aux;
  long long ld_aux;
  const float* resid;
  long long ld_resid;
  const int* row_map;
  float* out_f32;
  long long ld_o32;
  void* out_f16;
  long long ld_o16;
  float* col_sum;
  float* col_sumsq;
  const float* alpha_ptr;   // optional device scalar multiplied into alpha
  const float* row_scale;   // optional fp32 [m] factor applied with col_scale2 (after act)
  void* out_pre16;          // optional fp16 copy of the value before col_scale2 / row_scale / resid
  long long ld_pre16;
  const float* aux_scale;   // optional per-column affine applied to aux before the activation derivative
  const float* aux_shift;
  float* osum;              // optional: osum[c] += *osum_alpha * sum over rows of the rounded out_f16 values
  const float* osum_alpha;
  int pre_is_grad;          // GELU epilogue stores gelu'(v) through out_pre16 instead of v
};

__device__ __forceinline__ float gelu_erf(float x) { return fvit_gelu(x); }
__device__ __forceinline__ float gelu_erf_grad(float x) { return fvit_gelu_grad(x); }

__device__ __forceinline__ float load16_as_float(const void* base, long long idx, int bf16) {
  if (bf16) return __bfloat162float(reinterpret_cast<const __nv_bfloat16*>(base)[idx]);
  return __half2float(reinterpret_cast<const __half*>(base)[idx]);
}
__device__ __forceinline__ uint32_t pack2_16(float a, float b, int bf16) {
  if (bf16) {
    __nv_bfloat162 h = __floats2bfloat162_rn(a, b);
    return *reinterpret_cast<uint32_t*>(&h);
  }
  __half2 h = __floats2half2_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&h);
}

// 32-byte global accesses as two 16-byte vector accesses (one full sector per lane)
__device__ __forceinline__ void st_global_256(void* ptr, const uint32_t (&v)[8]) {
  uint4* q = reinterpret_cast<uint4*>(ptr);
  q[0] = make_uint4(v[0], v[1], v[2], v[3]);
  q[1] = make_uint4(v[4], v[5], v[6], v[7]);
}
__device__ __forceinline__ void ld_global_256(const void* ptr, uint32_t (&v)[8]) {
  const uint4* q = reinterpret_cast<const uint4*>(ptr);
  const uint4 a = q[0], b = q[1];
  v[0] = a.x, v[1] = a.y, v[2] = a.z, v[3] = a.w, v[4] = b.x, v[5] = b.y, v[6] = b.z, v[7] = b.w;
}
__device__ __forceinline__ float2 unpack2_16(uint32_t w, int bf16) {
  if (bf16) return __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&w));
  return __half22float2(*reinterpret_cast<const __half2*>(&w));
}

__device__ __forceinline__ float4 ld_vec4_guard(const float* p, int valid, float fill) {
  if (valid >= 4 && (reinterpret_cast<uintptr_t>(p) & 15) == 0) return __ldg(reinterpret_cast<const float4*>(p));
  float4 r = make_float4(fill, fill, fill, fill);
  if (valid > 0) r.x = __ldg(p);
  if (valid > 1) r.y = __ldg(p + 1);
  if (valid > 2) r.z = __ldg(p + 2);
  if (valid > 3) r.w = __ldg(p + 3);
  return r;
}
__device__ __forceinline__ void unpack4_16(uint2 pk, int bf16, float (&a)[4]) {
  if (bf16) {
    const __nv_bfloat162 lo = *reinterpret_cast<const __nv_bfloat162*>(&pk.x);
    const __nv_bfloat162 hi = *reinterpret_cast<const __nv_bfloat162*>(&pk.y);
    a[0] = __low2float(lo), a[1] = __high2float(lo), a[2] = __low2float(hi), a[3] = __high2float(hi);
  } else {
    const __half2 lo = *reinterpret_cast<const __half2*>(&pk.x);
    const __half2 hi = *reinterpret_cast<const __half2*>(&pk.y);
    a[0] = __low2float(lo), a[1] = __high2float(lo), a[2] = __low2float(hi), a[3] = __high2float(hi);
  }
}

// Sum 16 per-lane values over the 32 lanes of a warp with 16 shuffles (recursive halving).
// On return lane L (even lanes are the owners) holds in v[0] the total of column
// ((L>>4)&1)*8 + ((L>>3)&1)*4 + ((L>>2)&1)*2 + ((L>>1)&1).
__device__ __forceinline__ void warp_colsum16(float (&v)[16], int lane) {
#pragma unroll
  for (int width = 8, mask = 16; width >= 1; width >>= 1, mask >>= 1) {
    const bool upper = (lane & mask) != 0;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      if (i < width) {
        const float send = upper ? v[i] : v[i + width];
        const float keep = upper ? v[i + width] : v[i];
        v[i] = keep + __shfl_xor_sync(0xffffffffu, send, mask);
      }
    }
  }
  v[0] += __shfl_xor_sync(0xffffffffu, v[0], 1);
}
__device__ __forceinline__ int colsum16_owner_col(int lane) {
  return ((lane >> 4) & 1) * 8 + ((lane >> 3) & 1) * 4 + ((lane >> 2) & 1) * 2 + ((lane >> 1) & 1);
}

// Epilogue specialisation: GENERIC = every option decided at run time (backward modes, statistics,
// split-K atomics); otherwise ACT / RESID / O32 / O16 are compile-time and the unused paths vanish
// (the epilogue is instruction-issue bound, so this is worth ~2.5x on short-K tiles).
// FEAT: compile-time feature mask (the FVIT_GEMM_F_* bits of include/fvit.h); EF_GENERIC keeps every switch at run
// time.
enum : uint32_t {
  EF_GENERIC = FVIT_GEMM_F_GENERIC,
  EF_ACT_SHIFT = FVIT_GEMM_F_ACT_SHIFT,
  EF_RESID = FVIT_GEMM_F_RESID,
  EF_O32 = FVIT_GEMM_F_O32,
  EF_O16 = FVIT_GEMM_F_O16,
  EF_STATS = FVIT_GEMM_F_STATS,
  EF_PRE = FVIT_GEMM_F_PRE,
  EF_ATOMIC = FVIT_GEMM_F_ATOMIC,
  EF_ALPHAPTR = FVIT_GEMM_F_ALPHAPTR,
  EF_CS2 = FVIT_GEMM_F_CS2,
  EF_RS = FVIT_GEMM_F_RS,
  EF_OSUM = FVIT_GEMM_F_OSUM,        // per-column sum of the rounded 16-bit output (bias gradient of the next layer)
  EF_PREGRAD = FVIT_GEMM_F_PREGRAD,  // out_pre16 receives gelu'(v) (consumed by FVIT_ACT_MUL_AUX in the backward pass)
  EF_DIRECT = FVIT_GEMM_F_DIRECT,    // 16-bit outputs only: row-per-thread epilogue, 32-byte stores
};
// work unit -> (M tile, N tile, K split). Plain GEMMs keep the K splits of a tile adjacent; the tap-in-N mode
// walks all tiles of one K range first so concurrently running CTAs share the A / B slices in L2.
__device__ __forceinline__ void decode_work(const GemmParams& p, int w, int& tm, int& tn, int& split) {
  int t;
  if (p.b_ntaps > 1) {
    const int nt = p.tiles_m * p.tiles_n;
    split = w / nt;
    t = w - split * nt;
  } else {
    split = w % p.split_k;
    t = w / p.split_k;
  }
  tn = t % p.tiles_n;
  tm = t / p.tiles_n;
}

// Output columns [n0, n_end) of work unit tile tn (with taps in N: columns [tap * n, (tap + 1) * n) hold tap tap).
__device__ __forceinline__ void unit_cols(const GemmParams& p, int tn, int& n0, int& n_end) {
  n0 = tn * p.tile_n;
  n_end = min(p.n, n0 + p.tile_n);
  if (p.b_ntaps > 1) {
    const int tap = tn / p.tiles_per_tap;
    n0 = tap * p.n + (tn - tap * p.tiles_per_tap) * p.tile_n;
    n_end = min((tap + 1) * p.n, n0 + p.tile_n);
  }
}

// Main loop of one work unit for MMA width N: the MMA warpgroup g accumulates rows [64g, 64g + 64) of the tile
// over K blocks [kb0, kb1) and leaves them in the shared-memory accumulator tile. One K block's MMAs stay in flight
// while the next block's are issued; each warp releases a ring stage once its warpgroup's MMAs on it have completed.
// In slab mode a "K block" kb is (channel block kb / 9, tap kb % 9): A comes from the slab ring (a stage holds only
// the weight tile) and a slab is released with the stage of its third tap.
// The accumulator tile is written once the epilogue has released it (acc_empty of the previous unit, acc_parity =
// the parity of this CTA's unit count) and handed over through acc_full. Columns >= N of the tile keep the values
// of an earlier unit: the epilogue only reads the unit's valid columns.
template <int N, int TA, int TB, int BF16, bool SLAB>
__device__ __forceinline__ void gemm_mainloop(const GemmParams& p, uint8_t* smem, int stage_bytes, int a_stage_bytes,
                                              uint64_t* full_bar, uint64_t* empty_bar, int& stage, uint32_t& phase,
                                              uint8_t* slabs, uint64_t* slab_full, uint64_t* slab_empty, int& slab,
                                              uint32_t& slab_phase, int kb0, int kb1, float* accbuf,
                                              uint64_t* acc_full, uint64_t* acc_empty, uint32_t acc_parity) {
  const int g = (threadIdx.x >> 7) & 1;
  const int lane = threadIdx.x & 31;
  // K-major SW128: SBO = 1024 (8 rows x 128 B), LBO unused; MN-major SW128: LBO = BK*128 (next 64-wide MN atom),
  // SBO = 1024 (next 8 K rows). Rows 64..127 of A: 64 K-major rows on (8 KB) or the second 64-wide MN atom (8 KB).
  constexpr uint32_t a_lbo = TA ? BK * 128 : 16;
  constexpr uint32_t b_lbo = TB ? BK * 128 : 16;
  constexpr uint32_t a_kstep = TA ? MMA_K * 128 : MMA_K * 2;
  constexpr uint32_t b_kstep = TB ? MMA_K * 128 : MMA_K * 2;
  float d[N / 2];
#pragma unroll
  for (int i = 0; i < N / 2; ++i) d[i] = 0.f;
  int prev = -1;       // ring stage of the K block whose MMAs are still in flight
  int prev_slab = -1;  // slab mode: the slab to release with it (its third tap), or -1
  for (int kb = kb0; kb < kb1; ++kb) {
    uint32_t sa;
    int last_kb, done_slab = -1;
    if constexpr (SLAB) {
      const int dx = kb % 3;
      if (dx == 0) mbar_wait(&slab_full[slab], slab_phase);
      // rows 64g + dx .. of the slab (the swizzle phase follows the address: see make_smem_desc)
      sa = smem_u32(slabs + slab * SLAB_BYTES) + (64 * g + dx) * 128;
      last_kb = kb / 9 == p.kb_per_tap - 1;
      if (dx == 2) {
        done_slab = slab;
        if (++slab == SLAB_BUFS) {
          slab = 0;
          slab_phase ^= 1;
        }
      }
    } else {
      sa = smem_u32(smem + stage * stage_bytes) + g * 8192;
      last_kb = (kb + 1) % p.kb_per_tap == 0;
    }
    mbar_wait(&full_bar[stage], phase);
    const uint32_t sb = smem_u32(smem + stage * stage_bytes) + a_stage_bytes;
    auto mma = [&](int k) {
      Wgmma<N, TA, TB, BF16>::mma(d, make_smem_desc(sa + k * a_kstep, a_lbo, 1024, SWZ_128B),
                                  make_smem_desc(sb + k * b_kstep, b_lbo, 1024, SWZ_128B), 1u);
    };
    // a tap's last K-block is zero beyond kc (TMA out-of-bounds fill / zero-padded weights): its all-zero
    // 16-wide steps are not issued (K = 196 per conv tap: 13 instead of 16 MMAs; K = 784: 49 instead of 52)
    const int nk = last_kb ? p.k_tail16 : BK / MMA_K;
    // (each case is a complete wgmma group: a branch between the MMAs of one group would serialize them)
    switch (nk) {
      case 1: wgmma_fence(); mma(0); wgmma_commit(); break;
      case 2: wgmma_fence(); mma(0); mma(1); wgmma_commit(); break;
      case 3: wgmma_fence(); mma(0); mma(1); mma(2); wgmma_commit(); break;
      default: wgmma_fence(); mma(0); mma(1); mma(2); mma(3); wgmma_commit(); break;
    }
    wgmma_wait1();  // the previous K block's MMAs are complete
    if (prev >= 0) {
      __syncwarp();
      if (lane == 0) {
        mbar_arrive(&empty_bar[prev]);
        if (prev_slab >= 0) mbar_arrive(&slab_empty[prev_slab]);
      }
    }
    prev = stage;
    prev_slab = done_slab;
    if (++stage == p.stages) {
      stage = 0;
      phase ^= 1;
    }
  }
  wgmma_wait0();
  if (prev >= 0) {
    __syncwarp();
    if (lane == 0) {
      mbar_arrive(&empty_bar[prev]);
      if (prev_slab >= 0) mbar_arrive(&slab_empty[prev_slab]);
    }
  }
  mbar_wait(acc_empty, acc_parity ^ 1);  // the epilogue has read the previous unit's tile
  acc_store<N>(accbuf + g * 64 * ACC_LD, ACC_LD, d);
  mbar_arrive(acc_full);
}

template <int TA, int TB, int BF16, bool SLAB>
__device__ __forceinline__ void gemm_mainloop_n(int mma_n, const GemmParams& p, uint8_t* smem, int stage_bytes,
                                                int a_stage_bytes, uint64_t* full_bar, uint64_t* empty_bar, int& stage,
                                                uint32_t& phase, uint8_t* slabs, uint64_t* slab_full,
                                                uint64_t* slab_empty, int& slab, uint32_t& slab_phase, int kb0,
                                                int kb1, float* accbuf, uint64_t* acc_full, uint64_t* acc_empty,
                                                uint32_t acc_parity) {
#define FVIT_MAINLOOP(N)                                                                                          \
  gemm_mainloop<N, TA, TB, BF16, SLAB>(p, smem, stage_bytes, a_stage_bytes, full_bar, empty_bar, stage, phase, slabs,   \
                                 slab_full, slab_empty, slab, slab_phase, kb0, kb1, accbuf, acc_full, acc_empty, \
                                 acc_parity)
  switch (mma_n) {
    case 16: FVIT_MAINLOOP(16); break;
    case 32: FVIT_MAINLOOP(32); break;
    case 48: FVIT_MAINLOOP(48); break;
    case 64: FVIT_MAINLOOP(64); break;
    case 80: FVIT_MAINLOOP(80); break;
    case 96: FVIT_MAINLOOP(96); break;
    case 112: FVIT_MAINLOOP(112); break;
    default: FVIT_MAINLOOP(128); break;
  }
#undef FVIT_MAINLOOP
}

template <uint32_t FEAT>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
    gemm_wgmma_kernel(const __grid_constant__ CUtensorMap tmap_a,
                      const __grid_constant__ CUtensorMap tmap_b,
                      const __grid_constant__ GemmParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);  // SW128 atoms
  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;

  const int unit0 = blockIdx.x, nunits = gridDim.x;  // work units are dealt to CTAs round-robin
  // MN-major B is staged as whole 64-column atoms (the MMA reads the first columns of them)
  const int b_stage_bytes = (p.b_mn ? ((p.tile_n + 63) & ~63) : p.tile_n) * BK * 2;
  const int a_stage_bytes = p.slab_pitch ? 0 : A_STAGE_BYTES;  // slab mode: A lives in the slab ring
  const int stage_bytes = a_stage_bytes + b_stage_bytes;
  uint8_t* slabs = smem + p.stages * stage_bytes;  // (stage sizes are multiples of 2 KB: slabs stay 1024-aligned)
  uint8_t* ctrl = slabs + (p.slab_pitch ? SLAB_BUFS * SLAB_BYTES : 0);
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(ctrl);
  uint64_t* empty_bar = full_bar + MAX_STAGES;
  uint64_t* acc_full = empty_bar + MAX_STAGES;  // accumulator tile written (MMA warpgroups -> epilogue)
  uint64_t* acc_empty = acc_full + 1;           // accumulator tile read (epilogue -> MMA warpgroups)
  uint64_t* slab_full = acc_empty + 1;          // slab mode: slab loaded (producer -> MMA warpgroups)
  uint64_t* slab_empty = slab_full + SLAB_BUFS; // slab mode: slab's three taps done (MMA warps -> producer)
  float* accbuf = reinterpret_cast<float*>(ctrl + SMEM_CTRL_BYTES);

  if (warp == TMA_WARP && lane == 0) {
    tma_prefetch_desc(&tmap_a);
    tma_prefetch_desc(&tmap_b);
    for (int s = 0; s < p.stages; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], MMA_WARPS);  // one arrival per MMA warp
    }
    mbar_init(acc_full, MMA_THREADS);  // every thread arrives after its own accumulator stores
    mbar_init(acc_empty, EPI_THREADS);  // every thread arrives after its own accumulator reads
    for (int s = 0; s < SLAB_BUFS; ++s) {
      mbar_init(&slab_full[s], 1);
      mbar_init(&slab_empty[s], MMA_WARPS);
    }
    fence_mbar_init();
  }
  __syncthreads();

  const int work_total = p.tiles_m * p.tiles_n * p.split_k;

  if (warp >= TMA_WARP) {
    // ===================================================================== TMA producer
    setmaxnreg_dec<PRODUCER_REGS>();
    if (warp == TMA_WARP && lane == 0) {
      int stage = 0, slab = 0;
      uint32_t phase = 0, slab_phase = 0;
      for (int w = unit0; w < work_total; w += nunits) {
        int tm, tn, split;
        decode_work(p, w, tm, tn, split);
        const int m0 = tm * BM;
        int n0 = tn * p.tile_n;
        int b_shift = p.b_row_off;
        if (p.b_ntaps > 1) {
          const int tap = tn / p.tiles_per_tap;
          n0 = (tn - tap * p.tiles_per_tap) * p.tile_n;
          b_shift += p.tap_shift[tap];
        }
        const int kb0 = (int)((long long)p.num_kb * split / p.split_k);
        const int kb1 = (int)((long long)p.num_kb * (split + 1) / p.split_k);
        for (int kb = kb0; kb < kb1; ++kb) {
          if (p.slab_pitch) {
            // kb = 9 x channel block + 3 dy + dx; the slab of (channel block, dy) serves taps dx = 0, 1, 2
            const int dx = kb % 3, dy = kb / 3 % 3, kc0 = kb / 9 * BK;
            if (dx == 0) {
              mbar_wait(&slab_empty[slab], slab_phase ^ 1);
              mbar_expect_tx(&slab_full[slab], (uint32_t)SLAB_BYTES);
              tma_load_3d(slabs + slab * SLAB_BYTES, &tmap_a, &slab_full[slab], kc0,
                          m0 + (dy - 1) * p.slab_pitch - 1, p.tap_plane[0]);
            }
            mbar_wait(&empty_bar[stage], phase ^ 1);
            mbar_expect_tx(&full_bar[stage], (uint32_t)(p.tile_n * BK * 2));
            tma_load_2d(smem + stage * stage_bytes, &tmap_b, &full_bar[stage], ((3 * dy + dx) * p.kb_per_tap) * BK + kc0,
                        n0);
            if (dx == 2 && ++slab == SLAB_BUFS) {
              slab = 0;
              slab_phase ^= 1;
            }
            if (++stage == p.stages) {
              stage = 0;
              phase ^= 1;
            }
            continue;
          }
          mbar_wait(&empty_bar[stage], phase ^ 1);
          uint8_t* sa = smem + stage * stage_bytes;
          uint8_t* sb = sa + A_STAGE_BYTES;
          mbar_expect_tx(&full_bar[stage], (uint32_t)(A_STAGE_BYTES + (p.b_mn ? ((p.tile_n + 63) / 64) * BK * 128
                                                                               : p.tile_n * BK * 2)));
          if (!p.a_mn) {
            const int tap = kb / p.kb_per_tap;
            const int kc0 = (kb - tap * p.kb_per_tap) * BK;
            tma_load_3d(sa, &tmap_a, &full_bar[stage], kc0, m0 + p.tap_shift[tap], p.tap_plane[tap]);
          } else {
            // A stored [K rows][M cols]: two 64-wide MN atoms of BK rows each
            tma_load_3d(sa, &tmap_a, &full_bar[stage], m0, kb * BK + p.a_row_off, 0);
            tma_load_3d(sa + BK * 128, &tmap_a, &full_bar[stage], m0 + 64, kb * BK + p.a_row_off, 0);
          }
          if (!p.b_mn) {
            tma_load_2d(sb, &tmap_b, &full_bar[stage], kb * BK, n0);
          } else {
            for (int j = 0; j < (p.tile_n + 63) / 64; ++j)
              tma_load_2d(sb + j * BK * 128, &tmap_b, &full_bar[stage], n0 + j * 64, kb * BK + b_shift);
          }
          if (++stage == p.stages) {
            stage = 0;
            phase ^= 1;
          }
        }
      }
    }
  } else if (warp < MMA_WARPS) {
    // ===================================================================== MMA warpgroups
    int stage = 0, slab = 0;
    uint32_t phase = 0, slab_phase = 0;
    uint32_t acc_parity = 0;
    for (int w = unit0; w < work_total; w += nunits, acc_parity ^= 1) {
      int tm, tn, split_;
      decode_work(p, w, tm, tn, split_);
      int n0, n_end;
      unit_cols(p, tn, n0, n_end);
      const int mma_n = (n_end - n0 + 15) & ~15;  // a partial last N tile issues only its own columns
      const int kb0 = (int)((long long)p.num_kb * split_ / p.split_k);
      const int kb1 = (int)((long long)p.num_kb * (split_ + 1) / p.split_k);
#define FVIT_MAINLOOP_N(TA, TB, BF, SLAB)                                                                  \
  gemm_mainloop_n<TA, TB, BF, SLAB>(mma_n, p, smem, stage_bytes, a_stage_bytes, full_bar, empty_bar, stage, phase, slabs, \
                              slab_full, slab_empty, slab, slab_phase, kb0, kb1, accbuf, acc_full, acc_empty,     \
                              acc_parity)
      if ((FEAT & EF_GENERIC) && p.bf16) {
        if (p.slab_pitch) FVIT_MAINLOOP_N(0, 0, 1, true);
        else if (!p.a_mn && !p.b_mn) FVIT_MAINLOOP_N(0, 0, 1, false);
        else if (!p.a_mn) FVIT_MAINLOOP_N(0, 1, 1, false);
        else if (!p.b_mn) FVIT_MAINLOOP_N(1, 0, 1, false);
        else FVIT_MAINLOOP_N(1, 1, 1, false);
      } else {
        if (p.slab_pitch) FVIT_MAINLOOP_N(0, 0, 0, true);
        else if (!p.a_mn && !p.b_mn) FVIT_MAINLOOP_N(0, 0, 0, false);
        else if (!p.a_mn) FVIT_MAINLOOP_N(0, 1, 0, false);
        else if (!p.b_mn) FVIT_MAINLOOP_N(1, 0, 0, false);
        else FVIT_MAINLOOP_N(1, 1, 0, false);
      }
#undef FVIT_MAINLOOP_N
    }
  } else {
    // ===================================================================== epilogue warpgroup
    // Per work unit: wait for the accumulator tile, run the epilogue from it, release it. Warp w of the group owns
    // rows 32*w .. +32 of the tile and walks its 32-column chunks. Per chunk a warp
    //   1. issues its residual / aux global loads,
    //   2. reads the accumulators of its chunk from the shared-memory tile,
    //   3. works "coalesced": one instruction covers 4 rows x 128 contiguous bytes (8 lanes x float4
    //      per row), so residual loads and fp32 / fp16 stores are full-line accesses.
    setmaxnreg_inc<EPILOGUE_REGS>();
    const int quad = warp - MMA_WARPS;  // 32-row quarter of the tile this warp's epilogue covers
    const int et = threadIdx.x - MMA_THREADS;  // thread index within the epilogue warpgroup
    // per-CTA partial BatchNorm statistics (sum | sum of squares), flushed with one atomic per column at the end
    float* stat_s = reinterpret_cast<float*>(ctrl + SMEM_CTRL_BYTES + SMEM_ACC_BYTES);
    const int sub = lane >> 3;   // row within a 4-row group
    const int c4 = lane & 7;     // which float4 of the 32-column chunk
    constexpr bool GENERIC = (FEAT & EF_GENERIC) != 0;
    constexpr int ACT = (FEAT >> EF_ACT_SHIFT) & 7;
    const bool atomic_out = GENERIC ? (p.atomic_out != 0) : ((FEAT & EF_ATOMIC) != 0);
    const bool use_resid = GENERIC ? (p.resid != nullptr && !p.atomic_out) : ((FEAT & EF_RESID) != 0);
    const int act = GENERIC ? p.act : ACT;
    const bool use_aux = (act == FVIT_ACT_GELU_BWD || act == FVIT_ACT_RELU_BWD || act == FVIT_ACT_MUL_AUX) && !atomic_out;
    const bool out32 = GENERIC ? (p.out_f32 != nullptr) : ((FEAT & EF_O32) != 0);
    const bool out16 = GENERIC ? (p.out_f16 != nullptr) : ((FEAT & EF_O16) != 0);
    const bool stats = GENERIC ? (p.col_sum != nullptr && !p.atomic_out) : ((FEAT & EF_STATS) != 0);
    const bool has_cs2 = GENERIC ? (p.col_scale2 != nullptr) : ((FEAT & EF_CS2) != 0);
    const bool has_rs = GENERIC ? (p.row_scale != nullptr) : ((FEAT & EF_RS) != 0);
    const bool has_pre = GENERIC ? (p.out_pre16 != nullptr) : ((FEAT & EF_PRE) != 0);
    const bool pregrad = GENERIC ? (p.pre_is_grad != 0) : ((FEAT & EF_PREGRAD) != 0);
    const bool has_aptr = GENERIC ? (p.alpha_ptr != nullptr) : ((FEAT & EF_ALPHAPTR) != 0);
    const bool osum = GENERIC ? (p.osum != nullptr) : ((FEAT & EF_OSUM) != 0);
    const float alpha = has_aptr ? p.alpha * __ldg(p.alpha_ptr) : p.alpha;
    if (stats) {
      for (int i = et; i < 2 * p.n; i += EPI_THREADS) stat_s[i] = 0.f;
      asm volatile("bar.sync 1, %0;" ::"n"(EPI_THREADS) : "memory");  // the epilogue warps only
    }
    if (osum) {  // tile-local column sums: stat_s[0 .. tile_n)
      stat_s[et] = 0.f;
      asm volatile("bar.sync 1, %0;" ::"n"(EPI_THREADS) : "memory");
    }
    const float osum_alpha = (osum && p.osum_alpha) ? __ldg(p.osum_alpha) : 1.f;
    uint32_t acc_parity = 0;
    for (int w = unit0; w < work_total; w += nunits, acc_parity ^= 1) {
      int tm, tn, split_;
      decode_work(p, w, tm, tn, split_);
      const int row_base = tm * BM + quad * 32;
      int n0, n_end;
      unit_cols(p, tn, n0, n_end);
      // output rows of the 8 tile rows this lane touches (4k + sub), fetched once per tile (before the wait: row_map
      // reads do not depend on the accumulators)
      long long orow[8];
      {
        long long my_orow = -1;
        if (row_base + lane < p.m)
          my_orow = p.row_map ? (long long)p.row_map[row_base + lane] : (long long)(row_base + lane);
#pragma unroll
        for (int k = 0; k < 8; ++k) orow[k] = __shfl_sync(0xffffffffu, my_orow, 4 * k + sub);
      }
      mbar_wait(acc_full, acc_parity);

      const float* arow = accbuf + (quad * 32 + lane) * ACC_LD;  // this lane's accumulator row (row-per-thread reads)

      if constexpr ((FEAT & EF_DIRECT) != 0) {
        // Row-per-thread epilogue for launches that only write 16-bit outputs (qkv / fc1 / data gradients): lane l
        // owns tile row quad*32 + l, computes on 32 accumulator columns of its row and stores them as
        // two 32-byte sectors per output -- no staging tile, no per-row address math, one bounds check per 16 columns.
        // (n, the leading dimensions and the base pointers are multiples of 16 elements: checked by the launcher.)
        const int my_row = row_base + lane;
        const long long my_orow =
            my_row < p.m ? (p.row_map ? (long long)p.row_map[my_row] : (long long)my_row) : -1;
        uint16_t* const orow16 = reinterpret_cast<uint16_t*>(p.out_f16) + (my_orow >= 0 ? my_orow : 0) * p.ld_o16;
        uint16_t* const prow16 = reinterpret_cast<uint16_t*>(p.out_pre16) + (long long)my_row * p.ld_pre16;
        const uint16_t* const arow16 = reinterpret_cast<const uint16_t*>(p.aux) + (long long)my_row * p.ld_aux;
        for (int c0 = 0; c0 < p.tile_n; c0 += 32) {
          const int nbase = n0 + c0;
          if (nbase >= n_end) break;  // warp-uniform
          const int nvalid = min(min(32, n_end - nbase), p.tile_n - c0);   // 16 or 32
          uint32_t axw[2][8];
          if (use_aux && my_orow >= 0) {
            ld_global_256(arow16 + nbase, axw[0]);
            if (nvalid > 16) ld_global_256(arow16 + nbase + 16, axw[1]);
          }
          uint32_t raw[32];
#pragma unroll
          for (int i = 0; i < 8; ++i) {
            const float4 v = *reinterpret_cast<const float4*>(arow + c0 + 4 * i);
            raw[4 * i] = __float_as_uint(v.x), raw[4 * i + 1] = __float_as_uint(v.y);
            raw[4 * i + 2] = __float_as_uint(v.z), raw[4 * i + 3] = __float_as_uint(v.w);
          }
          float osv[32];  // rounded outputs for the column sums
#pragma unroll
          for (int hf = 0; hf < 2; ++hf) {
            if (hf * 16 >= nvalid) {
              if (osum) {
#pragma unroll
                for (int i = 0; i < 16; ++i) osv[hf * 16 + i] = 0.f;
              }
              continue;
            }
            const int col = nbase + hf * 16;
            uint32_t ow[8], pw[8];
#pragma unroll
            for (int q = 0; q < 4; ++q) {  // 4 columns at a time: per-column vectors are warp-uniform 16-byte loads
              float4 cs = make_float4(alpha, alpha, alpha, alpha), sh = make_float4(0.f, 0.f, 0.f, 0.f);
              if (p.col_scale) {
                const float4 t = __ldg(reinterpret_cast<const float4*>(p.col_scale + col) + q);
                cs.x *= t.x, cs.y *= t.y, cs.z *= t.z, cs.w *= t.w;
              }
              if (p.col_shift) sh = __ldg(reinterpret_cast<const float4*>(p.col_shift + col) + q);
              float v[4] = {fmaf(__uint_as_float(raw[hf * 16 + 4 * q]), cs.x, sh.x),
                            fmaf(__uint_as_float(raw[hf * 16 + 4 * q + 1]), cs.y, sh.y),
                            fmaf(__uint_as_float(raw[hf * 16 + 4 * q + 2]), cs.z, sh.z),
                            fmaf(__uint_as_float(raw[hf * 16 + 4 * q + 3]), cs.w, sh.w)};
              float pv[4] = {v[0], v[1], v[2], v[3]};
              if (act == FVIT_ACT_RELU) {
#pragma unroll
                for (int e = 0; e < 4; ++e) v[e] = fmaxf(v[e], 0.f);
              } else if (act == FVIT_ACT_GELU) {
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                  if (has_pre && pregrad) v[e] = fvit_gelu_both(v[e], pv[e]);
                  else v[e] = gelu_erf(v[e]);
                }
              }
              if (use_aux) {
                const float2 a01 = unpack2_16(axw[hf][2 * q], p.bf16), a23 = unpack2_16(axw[hf][2 * q + 1], p.bf16);
                float a[4] = {a01.x, a01.y, a23.x, a23.y};
                if (act == FVIT_ACT_MUL_AUX) {
#pragma unroll
                  for (int e = 0; e < 4; ++e) v[e] *= a[e];
                } else {
                  if (p.aux_scale) {
                    const float4 asc = __ldg(reinterpret_cast<const float4*>(p.aux_scale + col) + q);
                    const float4 ash = __ldg(reinterpret_cast<const float4*>(p.aux_shift + col) + q);
                    a[0] = fmaf(a[0], asc.x, ash.x), a[1] = fmaf(a[1], asc.y, ash.y), a[2] = fmaf(a[2], asc.z, ash.z),
                    a[3] = fmaf(a[3], asc.w, ash.w);
                  }
#pragma unroll
                  for (int e = 0; e < 4; ++e) {
                    if (act == FVIT_ACT_GELU_BWD) v[e] *= gelu_erf_grad(a[e]);
                    else v[e] = a[e] > 0.f ? v[e] : 0.f;
                  }
                }
              }
              ow[2 * q] = pack2_16(v[0], v[1], p.bf16), ow[2 * q + 1] = pack2_16(v[2], v[3], p.bf16);
              if (has_pre) pw[2 * q] = pack2_16(pv[0], pv[1], p.bf16), pw[2 * q + 1] = pack2_16(pv[2], pv[3], p.bf16);
              if (osum) {
                const float2 r01 = unpack2_16(ow[2 * q], p.bf16), r23 = unpack2_16(ow[2 * q + 1], p.bf16);
                const bool okr = my_orow >= 0;
                osv[hf * 16 + 4 * q] = okr ? r01.x : 0.f, osv[hf * 16 + 4 * q + 1] = okr ? r01.y : 0.f;
                osv[hf * 16 + 4 * q + 2] = okr ? r23.x : 0.f, osv[hf * 16 + 4 * q + 3] = okr ? r23.y : 0.f;
              }
            }
            if (my_orow >= 0) {
              st_global_256(orow16 + col, ow);
              if (has_pre) st_global_256(prow16 + col, pw);
            }
          }
          if (osum) {
            // column sums over the warp's 32 rows: butterfly that halves the live values per step; lane l ends
            // up with column c0 + l
#pragma unroll
            for (int sft = 16; sft >= 1; sft >>= 1) {
              const bool up = (lane & sft) != 0;
#pragma unroll
              for (int i = 0; i < sft; ++i) {
                const float send = up ? osv[i] : osv[i + sft];
                const float keep = up ? osv[i + sft] : osv[i];
                osv[i] = keep + __shfl_xor_sync(0xffffffffu, send, sft);
              }
            }
            if (lane < nvalid && osv[0] != 0.f) atomicAdd(stat_s + c0 + lane, osv[0]);
          }
        }
      } else
      for (int c0 = 0; c0 < p.tile_n; c0 += 32) {
        const int nbase = n0 + c0;
        if (nbase >= n_end) break;  // warp-uniform
        const int col = nbase + 4 * c4;            // first of this lane's 4 columns
        const bool cfull = col + 4 <= n_end;        // all 4 columns valid
        const bool cany = col < n_end;
        // ---- 1. global loads first
        float4 rv[8];
        uint2 av[8];
        if (use_resid) {
#pragma unroll
          for (int k = 0; k < 8; ++k) {
            rv[k] = make_float4(0.f, 0.f, 0.f, 0.f);
            if (cany && orow[k] >= 0) {
              const float* r = p.resid + orow[k] * p.ld_resid + col;
              if (cfull && p.vec_ok) {
                rv[k] = *reinterpret_cast<const float4*>(r);
              } else {
                rv[k].x = r[0];
                if (col + 1 < n_end) rv[k].y = r[1];
                if (col + 2 < n_end) rv[k].z = r[2];
                if (col + 3 < n_end) rv[k].w = r[3];
              }
            }
          }
        }
        if (use_aux) {
#pragma unroll
          for (int k = 0; k < 8; ++k) {
            av[k] = make_uint2(0u, 0u);
            if (cany && orow[k] >= 0) {
              const long long ab = (long long)(row_base + 4 * k + sub) * p.ld_aux + col;
              const uint16_t* ap = reinterpret_cast<const uint16_t*>(p.aux) + ab;
              if (cfull && p.vec_ok) {
                av[k] = *reinterpret_cast<const uint2*>(ap);
              } else {
                uint32_t e[4] = {0u, 0u, 0u, 0u};
#pragma unroll
                for (int i = 0; i < 4; ++i)
                  if (col + i < n_end) e[i] = ap[i];
                av[k] = make_uint2(e[0] | (e[1] << 16), e[2] | (e[3] << 16));
              }
            }
          }
        }
        float4 cs = make_float4(1.f, 1.f, 1.f, 1.f), sh = make_float4(0.f, 0.f, 0.f, 0.f),
               cs2 = make_float4(1.f, 1.f, 1.f, 1.f);
        if (cany) {
          if (p.col_scale) cs = ld_vec4_guard(p.col_scale + col, n_end - col, 1.f);
          if (p.col_shift) sh = ld_vec4_guard(p.col_shift + col, n_end - col, 0.f);
          if (has_cs2) cs2 = ld_vec4_guard(p.col_scale2 + col, n_end - col, 1.f);
        }
        cs.x *= alpha, cs.y *= alpha, cs.z *= alpha, cs.w *= alpha;  // fold alpha
        float4 asc = make_float4(1.f, 1.f, 1.f, 1.f), ash = make_float4(0.f, 0.f, 0.f, 0.f);
        if (use_aux && p.aux_scale && cany) {
          asc = ld_vec4_guard(p.aux_scale + col, n_end - col, 1.f);
          ash = ld_vec4_guard(p.aux_shift + col, n_end - col, 0.f);
        }
        // ---- 2./3. accumulators straight from the shared-memory tile; coalesced epilogue math + stores
        const float* stg = accbuf + (quad * 32) * ACC_LD + c0;
        float4 s1 = make_float4(0.f, 0.f, 0.f, 0.f), s2 = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
        for (int k = 0; k < 8; ++k) {
          const int rl = 4 * k + sub;  // row within the warp's 32
          const bool ok = cany && orow[k] >= 0;
          float4 v = *reinterpret_cast<const float4*>(stg + rl * ACC_LD + 4 * c4);
          if (atomic_out) {
            v.x *= alpha, v.y *= alpha, v.z *= alpha, v.w *= alpha;
            if (ok) {
              float* o = p.out_f32 + orow[k] * p.ld_o32 + col;
              if (cfull && p.vec_ok) {  // one 16-byte reduction instead of four (L2 atomic throughput bound)
                asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(o), "f"(v.x), "f"(v.y), "f"(v.z),
                             "f"(v.w)
                             : "memory");
              } else {
                atomicAdd(o, v.x);
                if (col + 1 < n_end) atomicAdd(o + 1, v.y);
                if (col + 2 < n_end) atomicAdd(o + 2, v.z);
                if (col + 3 < n_end) atomicAdd(o + 3, v.w);
              }
            }
            continue;
          }
          v.x = fmaf(v.x, cs.x, sh.x), v.y = fmaf(v.y, cs.y, sh.y), v.z = fmaf(v.z, cs.z, sh.z),
          v.w = fmaf(v.w, cs.w, sh.w);
          if (stats && ok) {
            s1.x += v.x, s1.y += v.y, s1.z += v.z, s1.w += v.w;
            s2.x += v.x * v.x, s2.y += v.y * v.y, s2.z += v.z * v.z, s2.w += v.w * v.w;
          }
          if (!ok) continue;
          float4 pv = v;  // what out_pre16 receives: the pre-activation value, or gelu'(v) with pre_is_grad
          if (act == FVIT_ACT_RELU) {
            v.x = fmaxf(v.x, 0.f), v.y = fmaxf(v.y, 0.f), v.z = fmaxf(v.z, 0.f), v.w = fmaxf(v.w, 0.f);
          } else if (act == FVIT_ACT_GELU) {
            if (has_pre && pregrad) {
              v.x = fvit_gelu_both(v.x, pv.x), v.y = fvit_gelu_both(v.y, pv.y), v.z = fvit_gelu_both(v.z, pv.z),
              v.w = fvit_gelu_both(v.w, pv.w);
            } else {
              v.x = gelu_erf(v.x), v.y = gelu_erf(v.y), v.z = gelu_erf(v.z), v.w = gelu_erf(v.w);
            }
          }
          if (has_pre) {
            uint16_t* o = reinterpret_cast<uint16_t*>(p.out_pre16) + (long long)(row_base + rl) * p.ld_pre16 + col;
            const uint32_t lo = pack2_16(pv.x, pv.y, p.bf16), hi = pack2_16(pv.z, pv.w, p.bf16);
            if (cfull && p.vec_ok) {
              *reinterpret_cast<uint2*>(o) = make_uint2(lo, hi);
            } else {
              o[0] = (uint16_t)(lo & 0xFFFF);
              if (col + 1 < n_end) o[1] = (uint16_t)(lo >> 16);
              if (col + 2 < n_end) o[2] = (uint16_t)(hi & 0xFFFF);
              if (col + 3 < n_end) o[3] = (uint16_t)(hi >> 16);
            }
          }
          if (act == FVIT_ACT_MUL_AUX) {
            float a[4];
            unpack4_16(av[k], p.bf16, a);
            v.x *= a[0], v.y *= a[1], v.z *= a[2], v.w *= a[3];
          } else if (use_aux) {
            float a[4];
            unpack4_16(av[k], p.bf16, a);
            if (p.aux_scale) {  // aux holds the raw convolution output: pre-activation = raw * scale + shift (BatchNorm)
              a[0] = fmaf(a[0], asc.x, ash.x), a[1] = fmaf(a[1], asc.y, ash.y), a[2] = fmaf(a[2], asc.z, ash.z),
              a[3] = fmaf(a[3], asc.w, ash.w);
            }
            if (act == FVIT_ACT_GELU_BWD) {
              v.x *= gelu_erf_grad(a[0]), v.y *= gelu_erf_grad(a[1]), v.z *= gelu_erf_grad(a[2]),
              v.w *= gelu_erf_grad(a[3]);
            } else {
              v.x = a[0] > 0.f ? v.x : 0.f, v.y = a[1] > 0.f ? v.y : 0.f, v.z = a[2] > 0.f ? v.z : 0.f,
              v.w = a[3] > 0.f ? v.w : 0.f;
            }
          }
          if (has_cs2) v.x *= cs2.x, v.y *= cs2.y, v.z *= cs2.z, v.w *= cs2.w;
          if (has_rs) {
            const float rs = __ldg(p.row_scale + row_base + rl);
            v.x *= rs, v.y *= rs, v.z *= rs, v.w *= rs;
          }
          if (use_resid) v.x += rv[k].x, v.y += rv[k].y, v.z += rv[k].z, v.w += rv[k].w;
          if (out32) {
            float* o = p.out_f32 + orow[k] * p.ld_o32 + col;
            if (cfull && p.vec_ok) {
              *reinterpret_cast<float4*>(o) = v;
            } else {
              o[0] = v.x;
              if (col + 1 < n_end) o[1] = v.y;
              if (col + 2 < n_end) o[2] = v.z;
              if (col + 3 < n_end) o[3] = v.w;
            }
          }
          if (out16) {
            uint16_t* o = reinterpret_cast<uint16_t*>(p.out_f16) + orow[k] * p.ld_o16 + col;
            const uint32_t lo = pack2_16(v.x, v.y, p.bf16), hi = pack2_16(v.z, v.w, p.bf16);
            if (cfull && p.vec_ok) {
              *reinterpret_cast<uint2*>(o) = make_uint2(lo, hi);
            } else {
              o[0] = (uint16_t)(lo & 0xFFFF);
              if (col + 1 < n_end) o[1] = (uint16_t)(lo >> 16);
              if (col + 2 < n_end) o[2] = (uint16_t)(hi & 0xFFFF);
              if (col + 3 < n_end) o[3] = (uint16_t)(hi >> 16);
            }
            if (osum) {
              float r4[4];
              unpack4_16(make_uint2(lo, hi), p.bf16, r4);
              s1.x += r4[0], s1.y += r4[1], s1.z += r4[2], s1.w += r4[3];
            }
          }
        }
        if (osum) {
#pragma unroll
          for (int o = 8; o <= 16; o <<= 1) {
            s1.x += __shfl_xor_sync(0xffffffffu, s1.x, o), s1.y += __shfl_xor_sync(0xffffffffu, s1.y, o);
            s1.z += __shfl_xor_sync(0xffffffffu, s1.z, o), s1.w += __shfl_xor_sync(0xffffffffu, s1.w, o);
          }
          if (sub == 0 && cany) {
            const int lc = c0 + 4 * c4;  // column within the tile
            atomicAdd(stat_s + lc, s1.x);
            if (col + 1 < n_end) atomicAdd(stat_s + lc + 1, s1.y);
            if (col + 2 < n_end) atomicAdd(stat_s + lc + 2, s1.z);
            if (col + 3 < n_end) atomicAdd(stat_s + lc + 3, s1.w);
          }
        }
        if (stats) {
          // lanes sharing c4 (lane, lane^8, lane^16, lane^24) hold partial sums of the same 4 columns
#pragma unroll
          for (int o = 8; o <= 16; o <<= 1) {
            s1.x += __shfl_xor_sync(0xffffffffu, s1.x, o), s1.y += __shfl_xor_sync(0xffffffffu, s1.y, o);
            s1.z += __shfl_xor_sync(0xffffffffu, s1.z, o), s1.w += __shfl_xor_sync(0xffffffffu, s1.w, o);
            s2.x += __shfl_xor_sync(0xffffffffu, s2.x, o), s2.y += __shfl_xor_sync(0xffffffffu, s2.y, o);
            s2.z += __shfl_xor_sync(0xffffffffu, s2.z, o), s2.w += __shfl_xor_sync(0xffffffffu, s2.w, o);
          }
          if (sub == 0 && cany) {
            atomicAdd(stat_s + col, s1.x), atomicAdd(stat_s + p.n + col, s2.x);
            if (col + 1 < n_end) atomicAdd(stat_s + col + 1, s1.y), atomicAdd(stat_s + p.n + col + 1, s2.y);
            if (col + 2 < n_end) atomicAdd(stat_s + col + 2, s1.z), atomicAdd(stat_s + p.n + col + 2, s2.z);
            if (col + 3 < n_end) atomicAdd(stat_s + col + 3, s1.w), atomicAdd(stat_s + p.n + col + 3, s2.w);
          }
        }
      }
      mbar_arrive(acc_empty);  // this thread's last read of the accumulator tile is done
      if (osum) {  // flush this tile's column sums: one global atomic per column per tile
        asm volatile("bar.sync 1, %0;" ::"n"(EPI_THREADS) : "memory");
        const int lc = et;
        if (lc < p.tile_n && n0 + lc < n_end) {
          const float a = stat_s[lc];
          if (a != 0.f) atomicAdd(p.osum + n0 + lc, a * osum_alpha);
        }
        stat_s[lc] = 0.f;
        asm volatile("bar.sync 1, %0;" ::"n"(EPI_THREADS) : "memory");
      }
    }
    if (stats) {
      asm volatile("bar.sync 1, %0;" ::"n"(EPI_THREADS) : "memory");
      for (int i = et; i < p.n; i += EPI_THREADS) {
        const float a = stat_s[i], b = stat_s[p.n + i];
        if (a != 0.f || b != 0.f) {
          atomicAdd(p.col_sum + i, a);
          atomicAdd(p.col_sumsq + i, b);
        }
      }
    }
  }
}

// ------------------------------------------------------------------------------------------ host
// Cost model of the tile width: the work units are dealt round-robin to min(units, SMs) persistent CTAs and the
// busiest CTA decides. A unit costs the MMA columns it issues (~ MMA time per K block; a partial last N tile issues
// its width rounded up to 16) plus a fixed part for the unit's A operand stream (16 KB per K block, the bytes of
// 128 B columns). The fixed part, 160 columns, is fitted to tile_n 32 / 64 / 96 / 128 timings of four linear shapes
// (M x N x K = 27136 x 784 x 784, 27136 x 3136 x 784, 27136 x 784 x 3136, 6272 x 1568 x 1568; fv4 levels 2 and 3) on
// an H100 SXM at 400 W; times relative to tile_n 128:
//   tile_n 32: 1.96 / 2.47 / 3.06 / 2.76   64: 1.27 / 1.39 / 1.56 / 1.61   96: 1.09 / 1.05 / 1.14 / 1.24
// Slab mode moves 17 KB of A per three taps instead of 16 KB per tap, and its per-column cost drops more than its
// per-unit cost: its fixed part, 140 columns, is fitted (least squares of the log time ratios) to tile_n 32 / 64 / 96
// / 128 timings of the two conv levels of fv4 at batch 128 (M x N x kc = 430592 x 196 x 196 and 115200 x 392 x 392,
// 9 taps; forward with BatchNorm statistics, data gradient * GELU', data gradient + residual) on an H100 SXM at 700 W;
// times relative to tile_n 128 (level 0 forward / dgrad, level 1 forward / dgrad):
//   tile_n 32: 2.52 / 2.46 / 2.33 / 2.29   64: 1.55 / 1.52 / 1.33 / 1.31   96: 1.41 / 1.38 / 1.01 / 1.01
// (The same shapes through per-tap boxes fit 88 columns: 2.23 / 2.20 / 2.04 / 2.01, 1.49 / 1.46 / 1.21 / 1.20,
// 1.41 / 1.41 / 1.00 / 0.99.)
// Units enumerate N tiles in decode_work's order. Cached per shape.
static int pick_tile_n(int m, int n, int split_k, int b_ntaps, bool slab, int sms) {
  const double kUnitFixed = slab ? 140.0 : 160.0;
  static std::mutex mu;
  static std::map<std::tuple<int, int, int, int, bool, int>, int> cache;
  const auto key = std::make_tuple(m, n, split_k, b_ntaps, slab, sms);
  std::lock_guard<std::mutex> lock(mu);
  auto it = cache.find(key);
  if (it != cache.end()) return it->second;
  int best = 32;
  double best_cost = 1e30;
  const int tiles_m = ceil_div(m, BM);
  for (int bn = 32; bn <= MAX_TILE_N; bn += 32) {
    const int tiles_per_tap = ceil_div(n, bn);
    const int tiles_n = tiles_per_tap * b_ntaps;
    const int tail = (n - (tiles_per_tap - 1) * bn + 15) & ~15;
    const long long nt = (long long)tiles_m * tiles_n;
    const long long work = nt * split_k;
    const int ctas = (int)(work < sms ? work : sms);
    double cost = 0.0;
    for (int c = 0; c < ctas; ++c) {
      double busy = 0.0;
      for (long long w = c; w < work; w += ctas) {
        const long long t = b_ntaps > 1 ? w % nt : w / split_k;  // as decode_work
        const int tn = (int)(t % tiles_n) % tiles_per_tap;      // N tile within its tap
        busy += (tn == tiles_per_tap - 1 ? tail : bn) + kUnitFixed;
      }
      cost = busy > cost ? busy : cost;
    }
    if (cost < best_cost - 1e-9) {
      best_cost = cost;
      best = bn;
    }
  }
  cache.emplace(key, best);
  return best;
}

// 3-D (or degenerate) 16-bit tensor map with a {b0, b1, 1} box, cached by geometry.
static int get_tmap(CUtensorMap* out, const void* base, uint64_t d0, uint64_t d1, uint64_t d2,
                    uint64_t s1_bytes, uint64_t s2_bytes, uint32_t b0, uint32_t b1, int rank) {
  uint64_t dims[3] = {d0, d1, d2};
  uint64_t strides[2] = {s1_bytes, s2_bytes};
  uint32_t box[3] = {b0, b1, 1};
  return cached_tmap_16bit(out, base, rank, dims, strides, box, CU_TENSOR_MAP_SWIZZLE_128B);
}

// The instantiated variants, one list for the launch table and for fvit_gemm_variants: the staging-tile epilogue
// masks, then the masks that also have a row-per-thread (EF_DIRECT) form.
#define FVIT_ACTF(x) ((uint32_t)(x) << EF_ACT_SHIFT)
#define FVIT_GEMM_STAGED_VARIANTS(X)                                                                  \
  /* inference / shared forward shapes */                                                            \
  X(FVIT_ACTF(0) | EF_O16)                                  /* qkv */                                \
  X(FVIT_ACTF(2) | EF_O16)                                  /* fc1, conv1 (eval) */                  \
  X(FVIT_ACTF(1) | EF_O16)                                  /* stem conv1 (eval) */                  \
  X(FVIT_ACTF(1) | EF_O32 | EF_O16)                         /* stem conv2 (eval) */                  \
  X(FVIT_ACTF(0) | EF_RESID | EF_O32)                       /* proj, fc2, conv dgrad */              \
  X(FVIT_ACTF(0) | EF_RESID | EF_O32 | EF_O16)              /* conv2 (eval) */                       \
  X(FVIT_ACTF(0) | EF_O32)                                  /* downsample, head */                   \
  X(FVIT_ACTF(0) | EF_O32 | EF_O16)                         /* downsample -> next level */           \
  /* training forward */                                                                             \
  X(FVIT_ACTF(0) | EF_O16 | EF_STATS)                       /* raw conv + BN statistics */           \
  X(FVIT_ACTF(2) | EF_O16 | EF_PRE)                         /* fc1 saving the pre-GELU value */      \
  X(FVIT_ACTF(2) | EF_O16 | EF_PRE | EF_PREGRAD)            /* fc1 saving gelu' */                   \
  X(FVIT_ACTF(0) | EF_RESID | EF_O32 | EF_RS)               /* branch + stochastic depth */          \
  X(FVIT_ACTF(0) | EF_RESID | EF_O32 | EF_CS2 | EF_PRE)     /* branch with layer scale */            \
  X(FVIT_ACTF(0) | EF_RESID | EF_O32 | EF_CS2 | EF_PRE | EF_RS)  /* layer scale + stochastic depth */ \
  /* backward */                                                                                     \
  X(FVIT_ACTF(0) | EF_O32 | EF_ATOMIC | EF_ALPHAPTR)        /* wgrad split-K */                      \
  X(FVIT_ACTF(0) | EF_O32 | EF_ALPHAPTR)                    /* wgrad single pass */                  \
  X(FVIT_ACTF(0) | EF_O16 | EF_ALPHAPTR)                    /* dgrad */                              \
  X(FVIT_ACTF(3) | EF_O16 | EF_ALPHAPTR)                    /* dgrad * gelu' */                      \
  X(FVIT_ACTF(3) | EF_O16)                                  /* conv dgrad * gelu' */                 \
  X(FVIT_ACTF(3) | EF_O16 | EF_ALPHAPTR | EF_OSUM)          /* fc2 dgrad * gelu' + fc1 bias grad */  \
  X(FVIT_ACTF(5) | EF_O16 | EF_ALPHAPTR)                    /* fc2 dgrad * saved gelu' */            \
  X(FVIT_ACTF(5) | EF_O16 | EF_ALPHAPTR | EF_OSUM)          /* ... + fc1 bias gradient */
#define FVIT_GEMM_DIRECT_VARIANTS(X)                         \
  X(FVIT_ACTF(0) | EF_O16)                                   \
  X(FVIT_ACTF(1) | EF_O16)                                   \
  X(FVIT_ACTF(2) | EF_O16)                                   \
  X(FVIT_ACTF(2) | EF_O16 | EF_PRE | EF_PREGRAD)             \
  X(FVIT_ACTF(0) | EF_O16 | EF_ALPHAPTR)                     \
  X(FVIT_ACTF(3) | EF_O16)                                   \
  X(FVIT_ACTF(5) | EF_O16 | EF_ALPHAPTR)                     \
  X(FVIT_ACTF(5) | EF_O16 | EF_ALPHAPTR | EF_OSUM)
#define FVIT_CASE(F) case (F):

// Argument validation and the kernel variant of one call: host only (no CUDA call, no device access), so the
// variant of a launch can be queried on a machine without a GPU.
static int select_variant(const fvit_gemm_args* a, uint32_t* variant) {
  FVIT_CHECK(a != nullptr, "fvit_gemm: null args");
  FVIT_CHECK(a->m > 0 && a->n > 0 && a->kc > 0, "fvit_gemm: bad dims m=%d n=%d kc=%d", a->m, a->n,
             a->kc);
  FVIT_CHECK(a->ntaps >= 1 && a->ntaps <= 16, "fvit_gemm: ntaps=%d out of range", a->ntaps);
  FVIT_CHECK(a->a && a->b, "fvit_gemm: null operand");
  FVIT_CHECK(a->lda % 8 == 0 && a->ldb % 8 == 0, "fvit_gemm: lda/ldb must be multiples of 8");
  FVIT_CHECK(!(a->a_mn_major && a->ntaps != 1), "fvit_gemm: taps need a K-major A operand");
  FVIT_CHECK(a->out_f32 || a->out_f16 || a->out_pre16, "fvit_gemm: no output");
  const int b_ntaps = a->b_ntaps > 1 ? a->b_ntaps : 1;
  if (b_ntaps > 1)
    FVIT_CHECK(b_ntaps <= 16 && a->a_mn_major && a->b_mn_major && a->ntaps == 1 && a->n % 4 == 0 && !a->col_sum,
               "fvit_gemm: b_ntaps needs MN-major A and B, ntaps == 1, n %% 4 == 0");
  const int split_k = a->split_k > 1 ? a->split_k : 1;
  if (split_k > 1)
    FVIT_CHECK(a->out_f32 && !a->out_f16 && !a->col_sum, "fvit_gemm: split_k needs out_f32 only");
  if (a->act == FVIT_ACT_GELU_BWD || a->act == FVIT_ACT_RELU_BWD || a->act == FVIT_ACT_MUL_AUX)
    FVIT_CHECK(a->aux != nullptr, "fvit_gemm: backward activation needs aux");
  FVIT_CHECK(a->act >= FVIT_ACT_NONE && a->act <= FVIT_ACT_MUL_AUX, "fvit_gemm: unknown activation code %d", a->act);
  FVIT_CHECK((a->col_sum == nullptr) == (a->col_sumsq == nullptr),
             "fvit_gemm: col_sum and col_sumsq go together");
  FVIT_CHECK(!a->col_sum || a->n <= STATS_MAX_N, "fvit_gemm: statistics support n <= %d", STATS_MAX_N);
  FVIT_CHECK((a->aux_scale == nullptr) == (a->aux_shift == nullptr), "fvit_gemm: aux_scale and aux_shift go together");
  FVIT_CHECK(!a->out_colsum || (a->out_f16 && !a->col_sum && split_k == 1 && b_ntaps == 1),
             "fvit_gemm: out_colsum needs out_f16, no BN statistics, no split-K");

  FVIT_CHECK(a->tile_n == 0 || (a->tile_n >= 16 && a->tile_n <= 256 && a->tile_n % 16 == 0),
             "fvit_gemm: tile_n=%d invalid", a->tile_n);
  FVIT_CHECK(a->cta_group >= 0 && a->cta_group <= 2, "fvit_gemm: cta_group=%d invalid", a->cta_group);

  // feature mask of this call: the matching specialisation if one was instantiated, else the generic kernel
  const bool atomic_out = split_k > 1;
  uint32_t feat = FVIT_ACTF(a->act);
  if (a->resid && !atomic_out) feat |= EF_RESID;
  if (a->out_f32) feat |= EF_O32;
  if (a->out_f16) feat |= EF_O16;
  if (a->col_sum) feat |= EF_STATS;
  if (a->out_pre16) feat |= EF_PRE;
  if (atomic_out) feat |= EF_ATOMIC;
  if (a->alpha_ptr) feat |= EF_ALPHAPTR;
  if (a->col_scale2) feat |= EF_CS2;
  if (a->row_scale) feat |= EF_RS;
  if (a->out_colsum) feat |= EF_OSUM;
  if (a->pre_is_grad && a->out_pre16 && a->act == FVIT_ACT_GELU) feat |= EF_PREGRAD;
  *variant = EF_GENERIC;
  if (a->bf16) return 0;  // bf16 operands: only the generic kernel instantiates their MMAs
  {
    // row-per-thread epilogue (EF_DIRECT): 16-bit outputs only, everything a lane touches in 32-byte pieces
    auto al32 = [](const void* q) { return (reinterpret_cast<uintptr_t>(q) & 31) == 0; };
    const uint32_t allowed = EF_O16 | EF_PRE | EF_PREGRAD | EF_ALPHAPTR | EF_OSUM | (7u << EF_ACT_SHIFT);
    const bool ok = (feat & ~allowed) == 0 && (feat & EF_O16) && b_ntaps == 1 && a->n % 16 == 0 &&
                    a->ld_out_f16 % 16 == 0 && al32(a->out_f16) &&
                    (!a->out_pre16 || (a->ld_out_pre16 % 16 == 0 && al32(a->out_pre16))) &&
                    (!a->aux || (a->ld_aux % 16 == 0 && al32(a->aux))) &&
                    (!a->col_scale || (reinterpret_cast<uintptr_t>(a->col_scale) & 15) == 0) &&
                    (!a->col_shift || (reinterpret_cast<uintptr_t>(a->col_shift) & 15) == 0) &&
                    (!a->aux_scale || ((reinterpret_cast<uintptr_t>(a->aux_scale) & 15) == 0 &&
                                       (reinterpret_cast<uintptr_t>(a->aux_shift) & 15) == 0));
    if (ok) {
      switch (feat) {  // the combinations with a direct specialisation
        FVIT_GEMM_DIRECT_VARIANTS(FVIT_CASE)
        feat |= EF_DIRECT;
        break;
        default:
          break;
      }
    }
  }
#define FVIT_DIRECT_CASE(F) case EF_DIRECT | (F):
  switch (feat) {
    FVIT_GEMM_STAGED_VARIANTS(FVIT_CASE)
    FVIT_GEMM_DIRECT_VARIANTS(FVIT_DIRECT_CASE)
    *variant = feat;
    break;
    default:
      break;
  }
#undef FVIT_DIRECT_CASE
  return 0;
}

}  // namespace fvit

extern "C" int fvit_gemm_variant(const fvit_gemm_args* a, uint32_t* variant) {
  FVIT_CHECK(variant != nullptr, "fvit_gemm_variant: null variant");
  return fvit::select_variant(a, variant);
}

extern "C" int fvit_gemm_variants(uint32_t* out, int cap) {
  using namespace fvit;
  int count = 0;
#define FVIT_LIST(F) \
  if (count < cap) out[count] = (F); \
  ++count;
#define FVIT_LIST_DIRECT(F) FVIT_LIST(EF_DIRECT | (F))
  FVIT_GEMM_STAGED_VARIANTS(FVIT_LIST)
  FVIT_GEMM_DIRECT_VARIANTS(FVIT_LIST_DIRECT)
#undef FVIT_LIST_DIRECT
#undef FVIT_LIST
  return count;
}

extern "C" int fvit_gemm(const fvit_gemm_args* a, void* stream) {
  using namespace fvit;
  uint32_t feat = 0;
  if (const int rc = select_variant(a, &feat)) return rc;
  const int b_ntaps = a->b_ntaps > 1 ? a->b_ntaps : 1;
  const int split_k = a->split_k > 1 ? a->split_k : 1;
  const int sms = num_sms();
  // a requested width above the widest MMA is split into two equal tiles (multiples of 16)
  const int num_kb = ceil_div(a->kc, BK) * a->ntaps;
  // slab mode: stride-1 3x3 taps on one plane, tap (dy, dx) shifted by (dy - 1) P + (dx - 1) rows. With one or two
  // K blocks per tap (kc <= 128) it was not faster on H100 (fv0's C = 64 / 128 levels: 0.98 ... 1.07x the time of
  // per-tap boxes), so those keep per-tap boxes.
  int slab_pitch = 0;
  if (a->ntaps == 9 && a->kc > 2 * BK && !a->a_mn_major && !a->b_mn_major && b_ntaps == 1 && split_k == 1) {
    const int P = a->tap_shift[7] - a->tap_shift[4];
    bool ok = P > 0;
    for (int t = 0; t < 9 && ok; ++t)
      ok = a->tap_plane[t] == a->tap_plane[0] && a->tap_shift[t] == (t / 3 - 1) * P + (t % 3 - 1);
    if (ok) slab_pitch = P;
  }
  int tile_n = a->tile_n > 0 ? a->tile_n
                             : pick_tile_n(a->m, a->n, split_k < num_kb ? split_k : num_kb, b_ntaps, slab_pitch > 0, sms);
  if (tile_n > MAX_TILE_N) tile_n = ceil_div(tile_n, 32) * 16;

  GemmParams p;
  memset(&p, 0, sizeof(p));
  p.m = a->m;
  p.n = a->n;
  p.kb_per_tap = ceil_div(a->kc, BK);
  p.num_kb = num_kb;
  {
    const int tail = a->kc - (p.kb_per_tap - 1) * BK;  // 1..64 real columns in the last block
    p.k_tail16 = ceil_div(tail, MMA_K);
  }
  p.a_mn = a->a_mn_major ? 1 : 0;
  p.b_mn = a->b_mn_major ? 1 : 0;
  p.a_row_off = a->a_row_off;
  p.b_row_off = a->b_row_off;
  p.tile_n = tile_n;
  p.tiles_m = ceil_div(a->m, BM);
  p.tiles_n = ceil_div(a->n, tile_n);
  p.b_ntaps = a->b_ntaps > 1 ? a->b_ntaps : 1;
  p.tiles_per_tap = p.tiles_n;
  p.tiles_n *= p.b_ntaps;
  p.split_k = split_k < p.num_kb ? split_k : p.num_kb;
  if (p.split_k < 1) p.split_k = 1;
  p.atomic_out = split_k > 1 ? 1 : 0;
  p.slab_pitch = slab_pitch;
  const int stage_bytes = (slab_pitch ? 0 : A_STAGE_BYTES) + (a->b_mn_major ? ((tile_n + 63) & ~63) : tile_n) * BK * 2;
  const int slab_bytes = slab_pitch ? SLAB_BUFS * SLAB_BYTES : 0;
  const int stats_bytes = a->col_sum ? SMEM_STATS_BYTES : (a->out_colsum ? 256 * 4 : 0);
  int stages =
      (SMEM_BUDGET - SMEM_CTRL_BYTES - SMEM_ALIGN_SLACK - SMEM_ACC_BYTES - stats_bytes - slab_bytes) / stage_bytes;
  if (stages > MAX_STAGES) stages = MAX_STAGES;
  FVIT_CHECK(stages >= 2, "fvit_gemm: not enough shared memory for 2 stages");
  p.stages = stages;
  for (int i = 0; i < 16; ++i) {
    p.tap_shift[i] = i < (b_ntaps > 1 ? b_ntaps : a->ntaps) ? a->tap_shift[i] : 0;
    p.tap_plane[i] = i < a->ntaps ? a->tap_plane[i] : 0;
  }
  p.alpha = a->alpha;
  p.act = a->act;
  p.bf16 = a->bf16 ? 1 : 0;
  p.col_scale = a->col_scale;
  p.col_shift = a->col_shift;
  p.col_scale2 = a->col_scale2;
  p.aux = a->aux;
  p.ld_aux = a->ld_aux;
  p.resid = a->resid;
  p.ld_resid = a->ld_resid;
  p.row_map = a->row_map;
  p.out_f32 = a->out_f32;
  p.ld_o32 = a->ld_out_f32;
  p.out_f16 = a->out_f16;
  p.ld_o16 = a->ld_out_f16;
  p.col_sum = a->col_sum;
  p.col_sumsq = a->col_sumsq;
  p.alpha_ptr = a->alpha_ptr;
  p.row_scale = a->row_scale;
  p.out_pre16 = a->out_pre16;
  p.ld_pre16 = a->ld_out_pre16;
  p.aux_scale = a->aux_scale;
  p.aux_shift = a->aux_shift;
  p.osum = a->out_colsum;
  p.osum_alpha = a->out_colsum_alpha;
  p.pre_is_grad = (a->pre_is_grad && a->out_pre16 && a->act == FVIT_ACT_GELU) ? 1 : 0;
  // vector path: every touched row segment must be 16-byte aligned
  bool vec = true;
  if (a->out_f32)
    vec = vec && (a->ld_out_f32 % 4 == 0) && ((reinterpret_cast<uintptr_t>(a->out_f32) & 15) == 0);
  if (a->out_f16)
    vec = vec && (a->ld_out_f16 % 8 == 0) && ((reinterpret_cast<uintptr_t>(a->out_f16) & 15) == 0);
  if (a->resid)
    vec = vec && (a->ld_resid % 4 == 0) && ((reinterpret_cast<uintptr_t>(a->resid) & 15) == 0);
  if (a->out_pre16)
    vec = vec && (a->ld_out_pre16 % 4 == 0) && ((reinterpret_cast<uintptr_t>(a->out_pre16) & 7) == 0);
  if (a->aux)
    vec = vec && (a->ld_aux % 4 == 0) && ((reinterpret_cast<uintptr_t>(a->aux) & 7) == 0);
  p.vec_ok = vec ? 1 : 0;
  CUtensorMap tma, tmb;
  int rc;
  if (!p.a_mn) {
    const int planes = a->a_planes > 0 ? a->a_planes : 1;
    rc = get_tmap(&tma, a->a, (uint64_t)a->kc, (uint64_t)a->a_rows, (uint64_t)planes,
                  (uint64_t)a->lda * 2,
                  (uint64_t)(planes > 1 ? a->a_plane_stride : a->a_rows * a->lda) * 2, BK,
                  slab_pitch ? SLAB_ROWS : BM, 3);
  } else {
    rc = get_tmap(&tma, a->a, (uint64_t)a->m, (uint64_t)a->a_rows, 1, (uint64_t)a->lda * 2,
                  (uint64_t)a->a_rows * a->lda * 2, 64, BK, 3);
  }
  if (rc) return rc;
  if (!p.b_mn) {
    const uint64_t kdim = a->ntaps == 1 ? (uint64_t)a->kc : (uint64_t)p.num_kb * BK;
    rc = get_tmap(&tmb, a->b, kdim, (uint64_t)a->n, 1, (uint64_t)a->ldb * 2, 0, BK,
                  (uint32_t)tile_n, 2);
  } else {
    rc = get_tmap(&tmb, a->b, (uint64_t)a->n, (uint64_t)a->b_rows, 1, (uint64_t)a->ldb * 2, 0, 64,
                  BK, 2);
  }
  if (rc) return rc;

  const int smem_bytes =
      stages * stage_bytes + slab_bytes + SMEM_CTRL_BYTES + SMEM_ALIGN_SLACK + SMEM_ACC_BYTES + stats_bytes;
  const long long work = (long long)p.tiles_m * p.tiles_n * p.split_k;
  const int grid = (int)(work < sms ? work : sms);
#define FVIT_GEMM_LAUNCH(F)                                                                          \
  do {                                                                                               \
    auto kfn = gemm_wgmma_kernel<(F)>;                                                               \
    static bool attr_set = false;                                                                    \
    if (!attr_set) {                                                                                 \
      FVIT_CUDA(cudaFuncSetAttribute(kfn, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BUDGET)); \
      attr_set = true;                                                                               \
    }                                                                                                \
    kfn<<<grid, GEMM_THREADS, smem_bytes, (cudaStream_t)stream>>>(tma, tmb, p);                      \
    return post_launch("gemm_wgmma_kernel");                                                         \
  } while (0)
#define FVIT_LAUNCH_CASE(F) \
  case (F):                 \
    FVIT_GEMM_LAUNCH(F);
#define FVIT_LAUNCH_DIRECT_CASE(F) FVIT_LAUNCH_CASE(EF_DIRECT | (F))
  switch (feat) {
    FVIT_GEMM_STAGED_VARIANTS(FVIT_LAUNCH_CASE)
    FVIT_GEMM_DIRECT_VARIANTS(FVIT_LAUNCH_DIRECT_CASE)
    default:
      break;
  }
  FVIT_GEMM_LAUNCH(EF_GENERIC);
#undef FVIT_LAUNCH_DIRECT_CASE
#undef FVIT_LAUNCH_CASE
#undef FVIT_GEMM_LAUNCH
}
