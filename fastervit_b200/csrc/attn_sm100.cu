// fvit_attn_tc_fwd: tensor-core attention core of WindowAttention.forward (fv.py:559-565) for sm_90a.
//
// Work item = (tile of 128 consecutive token rows, head). A tile holds gpt = floor(128 / S) whole
// windows (groups of S tokens: ct_size^2 carrier tokens + ws^2 window tokens, or the carrier grid of
// one image); rows of the box beyond gpt*S belong to the next tile and are masked.
//
//   warp 4     : TMA producer — Q, K, V head slices (128 x hdp, 16-bit) of the packed qkv matrix into
//                a ring of swizzled shared-memory head tiles (attn_head.cuh: hdp 32, 64 or 80)
//   warps 0..3 : one warpgroup — S = Q K^T (wgmma, M=128 as two m64 halves, N=128, K=hdp) into an fp32
//                score tile in shared memory; softmax with one thread per query row: block-diagonal
//                window mask, relative-position bias from shared memory, fp32 max / exp2 / sum, P written
//                as fp16 straight into the 128B-swizzled operand layout; O = P V (B = V as an MN-major
//                operand, N = hdp) into the same tile; then the O epilogue (1/rowsum, fp16, 16-byte stores).
// Scores and probabilities never touch HBM; per row the kernel reads 3*hdp*2 B and writes hdp*2 B.
#include <cuda_fp16.h>

#include <mutex>
#include <unordered_map>

#include "../../include/fvit.h"
#include "attn_head.cuh"
#include "common.h"
#include "ptx.cuh"

namespace fvit {

constexpr int AT_THREADS = 160;
constexpr int AT_ROWS = 128;
constexpr int AT_PRODUCER = 4;           // the TMA warp; warps 0..3 are the compute warpgroup
constexpr int AT_ACC_LD = 132;           // floats per row of the fp32 accumulator tile (conflict-free float4 rows)
constexpr int AT_ACC_BYTES = AT_ROWS * AT_ACC_LD * 4;

struct AttnParams {
  int groups, S, heads, gpt, tiles;
  int slot;  // rows per window slot inside the 128-row tile: smallest of {16, 32, 64, 128} >= S
  int rows_total;
  float scale_log2e;
  const float* bias;  // [heads, S, S] or null
  __half* out;
  long long ldo;
};

template <int HDP>
struct AttnSmem {
  static constexpr int NST = HDP == 32 ? 2 : 1;              // Q/K/V ring depth
  static constexpr int TILE_BYTES = AT_ROWS * HDP * 2;       // one of Q / K / V
  static constexpr int STAGE_BYTES = 3 * TILE_BYTES;
  static constexpr int P_BYTES = AT_ROWS * 128 * 2;          // 128 x 128 fp16, two 64-wide K atoms
  static constexpr int P_OFF = NST * STAGE_BYTES;
  static constexpr int ACC_OFF = P_OFF + P_BYTES;
  static constexpr int BIAS_OFF = ACC_OFF + AT_ACC_BYTES;
};

// Window w of a tile lives in rows [w*slot, w*slot + S) of the 128-row operand tiles (slot = 16/32/64/
// 128), so a query row only ever meets the keys of its own slot: the S x S diagonal blocks of the
// 128 x 128 score matrix. Rows >= S of a slot hold the first rows of the next window (harmless:
// masked as keys, not written as queries).
template <int HDP>
__global__ void __launch_bounds__(AT_THREADS, 1)
    attn_tc_kernel(const __grid_constant__ CUtensorMap tmap_qkv, const __grid_constant__ CUtensorMap tmap_qkv_b,
                   const __grid_constant__ AttnParams p) {
  using SM = AttnSmem<HDP>;
  using HT = HeadTile<HDP>;
  constexpr int NST = SM::NST;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int S = p.S;
  float* bias_s = reinterpret_cast<float*>(smem + SM::BIAS_OFF);
  float* acc = reinterpret_cast<float*>(smem + SM::ACC_OFF);
  uint8_t* ctrl = smem + SM::BIAS_OFF + ((S * S * 4 + 15) & ~15);
  uint64_t* qkv_full = reinterpret_cast<uint64_t*>(ctrl);  // [2]
  uint64_t* qkv_empty = qkv_full + 2;                      // [2]

  if (warp == AT_PRODUCER && lane == 0) {
    tma_prefetch_desc(&tmap_qkv);
    if (HT::HB > 0) tma_prefetch_desc(&tmap_qkv_b);
    for (int i = 0; i < 2; ++i) {
      mbar_init(&qkv_full[i], 1);
      mbar_init(&qkv_empty[i], 1);
    }
    fence_mbar_init();
  }
  __syncthreads();

  const int items = p.tiles * p.heads;
  const int nslots = AT_ROWS / p.slot;

  if (warp == AT_PRODUCER) {
    if (lane == 0) {
      int it = 0;
      for (int w = blockIdx.x; w < items; w += gridDim.x, ++it) {
        const int st = it % NST;
        const uint32_t ph = (it / NST) & 1;
        const int head = w / p.tiles, tile = w % p.tiles;  // head-major: bias is re-staged rarely
        mbar_wait(&qkv_empty[st], ph ^ 1);
        uint8_t* base = smem + st * SM::STAGE_BYTES;
        mbar_expect_tx(&qkv_full[st], SM::STAGE_BYTES);
        for (int sl = 0; sl < nslots; ++sl) {
          // window (tile*gpt + sl) -> rows [sl*slot, (sl+1)*slot) of the three operand tiles; windows
          // past the end give out-of-range rows, which TMA zero-fills
          const int row0 = (tile * p.gpt + sl) * S;
          for (int op = 0; op < 3; ++op)
            HT::load(base + op * SM::TILE_BYTES, AT_ROWS, sl * p.slot, &tmap_qkv, &tmap_qkv_b, &qkv_full[st],
                     (op * p.heads + head) * HDP, row0);
        }
      }
    }
  } else {
    // ------------------------------------------------------------------ MMA + softmax + epilogue warpgroup
    const int quad = warp & 3;
    const int r = quad * 32 + lane;    // row in tile
    const int tid = threadIdx.x;       // 0..127
    const int slot = p.slot;
    const int sl = r / slot;           // window slot of this row
    const int j = r - sl * slot;       // token index inside the window
    const int lo = sl * slot;          // first key column of the window
    // key columns of the warp's rows: slots are >= 32 rows or the warp spans 32/slot whole slots
    const int wlo = slot >= 32 ? lo : quad * 32;
    const int wn = slot >= 32 ? S : 32;            // columns to visit starting at wlo
    const int nch = (wn + 31) / 32;
    uint8_t* sP = smem + SM::P_OFF;
    const uint32_t sP_u = smem_u32(sP);
    const float* arow = acc + r * AT_ACC_LD;
    // columns outside [wlo, wlo + 32*nch) are never written by this warp's rows: zero them once
    for (int c = 0; c < 128; c += 8) {
      if (c + 8 <= wlo || c >= wlo + 32 * nch)
        *reinterpret_cast<uint4*>(sP + (c >> 6) * (AT_ROWS * 128) + r * 128 + ((((c & 63) >> 3) ^ (r & 7)) << 4)) =
            make_uint4(0, 0, 0, 0);
    }
    int it = 0;
    int staged_head = -1;
    for (int w = blockIdx.x; w < items; w += gridDim.x, ++it) {
      const int st = it % NST;
      const uint32_t ph = (it / NST) & 1;
      const int head = w / p.tiles, tile = w % p.tiles;
      const int grp = tile * p.gpt + sl;
      const bool row_ok = j < S && sl < p.gpt && grp < p.groups;
      // stage this head's bias (pre-multiplied by log2 e) in shared memory when the head changes;
      // loads are issued in batches of 8 so their latencies overlap
      if (p.bias && head != staged_head) {
        named_bar_sync(1, 128);  // previous head's readers are done
        const float* bsrc = p.bias + (long long)head * S * S;
        const int n = S * S;
        for (int i0 = tid; i0 < n; i0 += 128 * 8) {
          float tmp[8];
#pragma unroll
          for (int u = 0; u < 8; ++u) {
            const int i = i0 + u * 128;
            tmp[u] = i < n ? __ldg(bsrc + i) : 0.f;
          }
#pragma unroll
          for (int u = 0; u < 8; ++u) {
            const int i = i0 + u * 128;
            if (i < n) bias_s[i] = tmp[u] * 1.4426950408889634f;
          }
        }
        named_bar_sync(1, 128);
        staged_head = head;
      }

      mbar_wait(&qkv_full[st], ph);
      const uint32_t sQ = smem_u32(smem + st * SM::STAGE_BYTES);
      const uint32_t sK = sQ + SM::TILE_BYTES;
      const uint32_t sV = sQ + 2 * SM::TILE_BYTES;
      named_bar_sync(1, 128);  // the previous item's O reads of the accumulator tile are done
      wg_mma_128<128, 0, 0, HT::KSTEPS>(
          acc, AT_ACC_LD, [&](int h, int k) { return HT::kdesc(sQ, AT_ROWS, h * 64, k); },
          [&](int k) { return HT::kdesc(sK, AT_ROWS, 0, k); }, false);
      named_bar_sync(1, 128);
      // brow[c - lo] = bias of (this row, key c); rows that are not real queries read row 0 (unused)
      const float* brow = bias_s + (row_ok ? j : 0) * S;
      const bool use_bias = p.bias != nullptr;
      // pass 1: row maximum over the window's keys
      float mx = -INFINITY;
      for (int ch = 0; ch < nch; ++ch) {
        const int c0 = wlo + 32 * ch;
        uint32_t raw[32];
        ld_row32(arow + c0, raw);
#pragma unroll
        for (int u = 0; u < 32; ++u) {
          const int kk = c0 + u - lo;               // key index inside the window
          const bool in = kk >= 0 && kk < S;
          const float b = use_bias ? brow[in ? kk : 0] : 0.f;
          const float sc = fmaf(__uint_as_float(raw[u]), p.scale_log2e, b);
          mx = fmaxf(mx, in ? sc : -INFINITY);
        }
      }
      if (!row_ok) mx = 0.f;
      // pass 2: probabilities (unnormalised) -> fp16 operand tile, row sum
      float sum = 0.f;
      for (int ch = 0; ch < nch; ++ch) {
        const int c0 = wlo + 32 * ch;
        uint32_t raw[32];
        ld_row32(arow + c0, raw);
        uint32_t pk[16];
#pragma unroll
        for (int u = 0; u < 32; u += 2) {
          float e[2];
#pragma unroll
          for (int t = 0; t < 2; ++t) {
            const int kk = c0 + u + t - lo;
            const bool in = row_ok && kk >= 0 && kk < S;
            const float b = use_bias ? brow[in ? kk : 0] : 0.f;
            const float sc = fmaf(__uint_as_float(raw[u + t]), p.scale_log2e, b - mx);
            e[t] = in ? exp2f(sc) : 0.f;
          }
          const __half2 h = __floats2half2_rn(e[0], e[1]);
          // accumulate what the tensor core will actually multiply (fp16-rounded probabilities)
          sum += __low2float(h) + __high2float(h);
          pk[u >> 1] = *reinterpret_cast<const uint32_t*>(&h);
        }
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const int c = c0 + q * 8;
          if (c < 128)
            *reinterpret_cast<uint4*>(sP + (c >> 6) * (AT_ROWS * 128) + r * 128 +
                                      ((((c & 63) >> 3) ^ (r & 7)) << 4)) =
                make_uint4(pk[4 * q], pk[4 * q + 1], pk[4 * q + 2], pk[4 * q + 3]);
        }
      }
      // P is complete: publish it to the async proxy; every score read is done before O overwrites the tile
      fence_proxy_async_smem();
      named_bar_sync(1, 128);
      wg_mma_128_head<HDP, 0, 8>(
          acc, AT_ACC_LD,  // 128 keys in steps of 16
          [&](int h, int ks) {
            return make_smem_desc(sP_u + (ks >> 2) * (AT_ROWS * 128) + h * 64 * 128 + (ks & 3) * 32, 16, 1024, SWZ_128B);
          },
          sV, AT_ROWS, false);
      named_bar_sync(1, 128);
      if (tid == 0) mbar_arrive(&qkv_empty[st]);  // Q / K / V of this stage are consumed
      const float inv = row_ok ? 1.f / sum : 0.f;
      const long long grow = (long long)grp * S + j;
      if (row_ok) store_row_f16<HDP>(arow, inv, p.out + grow * p.ldo + head * HDP);
    }
  }
}

template <int HDP>
static int launch_attn(const CUtensorMap& tm, const CUtensorMap& tmb, const AttnParams& p, cudaStream_t st) {
  const size_t smem = 1024 + AttnSmem<HDP>::BIAS_OFF + ((size_t)p.S * p.S * 4 + 15) / 16 * 16 + 128;
  FVIT_CHECK(smem <= 227 * 1024, "fvit_attn_tc_fwd: needs %zu B of shared memory", smem);
  static bool configured = false;
  if (!configured) {
    FVIT_CUDA(cudaFuncSetAttribute(attn_tc_kernel<HDP>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
    configured = true;
  }
  const int items = p.tiles * p.heads;
  const int slots = num_sms();
  attn_tc_kernel<HDP><<<items < slots ? items : slots, AT_THREADS, smem, st>>>(tm, tmb, p);
  return post_launch("attn_tc_kernel");
}

}  // namespace fvit

using namespace fvit;

extern "C" int fvit_attn_tc_fwd(const void* qkv, int64_t ldq, int32_t groups, int32_t S, int32_t heads,
                                int32_t hdp, const float* bias, float scale, void* out, int64_t ldo,
                                void* stream) {
  FVIT_CHECK(qkv && out && groups > 0 && heads > 0, "fvit_attn_tc_fwd: bad arguments");
  FVIT_CHECK(S >= 1 && S <= 128, "fvit_attn_tc_fwd: S=%d unsupported (1..128)", S);
  FVIT_CHECK(hdp == 32 || hdp == 64 || hdp == 80, "fvit_attn_tc_fwd: padded head dim %d unsupported (32, 64 or 80)",
             hdp);
  FVIT_CHECK(ldq % 8 == 0 && ldo % 8 == 0 && ldq >= 3 * heads * hdp && ldo >= heads * hdp,
             "fvit_attn_tc_fwd: bad leading dimensions");
  FVIT_CHECK((reinterpret_cast<uintptr_t>(out) & 15) == 0, "fvit_attn_tc_fwd: out must be 16-byte aligned");
  AttnParams p;
  p.groups = groups;
  p.S = S;
  p.heads = heads;
  p.slot = S <= 16 ? 16 : (S <= 32 ? 32 : (S <= 64 ? 64 : 128));
  p.gpt = AT_ROWS / p.slot;
  p.tiles = (groups + p.gpt - 1) / p.gpt;
  p.rows_total = groups * S;
  p.scale_log2e = scale * 1.4426950408889634f;
  p.bias = bias;
  p.out = (__half*)out;
  p.ldo = ldo;
  CUtensorMap tm, tmb;
  int rc = head_tile_tmaps(&tm, &tmb, qkv, 3 * heads * hdp, p.rows_total, ldq, hdp, p.slot);
  if (rc) return rc;
  if (hdp == 80) return launch_attn<80>(tm, tmb, p, (cudaStream_t)stream);
  if (hdp == 64) return launch_attn<64>(tm, tmb, p, (cudaStream_t)stream);
  return launch_attn<32>(tm, tmb, p, (cudaStream_t)stream);
}

// =====================================================================================================
// fvit_attn_tc_bwd: tensor-core backward of the attention core for S <= 64 (window slots of 16/32/64 rows).
//   S  = Q K^T, dP = dO V^T                     (wgmma, 128x128 each, in turn in one fp32 shared-memory tile)
//   per query row (one thread each): P = softmax(S*scale + bias), delta = sum_c P*dP, dS = P*(dP - delta);
//       P and dS written as fp16 into two 128x128 swizzled operand tiles; dS accumulated into a per-CTA
//       shared-memory copy of dbias[head] (flushed with global atomics when the head changes)
//   dV = P^T dO, dK = dS^T Q (A = the tile read MN-major), dQ = dS K   -> the same tile, scaled, stored fp16.
// Scores / probabilities never touch HBM; per row the kernel reads 4*hdp*2 B and writes 3*hdp*2 B.
namespace fvit {

struct AttnBwdParams {
  int groups, S, heads, gpt, tiles, slot, hd;
  float scale, scale_log2e;
  const float* bias;
  float* dbias;
  __half* dqkv;
  long long lddq;
};

template <int HDP>
__global__ void __launch_bounds__(AT_THREADS, 1)
    attn_bwd_tc_kernel(const __grid_constant__ CUtensorMap tmap_qkv, const __grid_constant__ CUtensorMap tmap_do,
                       const __grid_constant__ CUtensorMap tmap_qkv_b, const __grid_constant__ CUtensorMap tmap_do_b,
                       const __grid_constant__ AttnBwdParams p) {
  using HT = HeadTile<HDP>;
  constexpr int TILE_BYTES = AT_ROWS * HDP * 2;
  constexpr int STAGE_BYTES = 4 * TILE_BYTES;  // Q, K, V, dO
  constexpr int NST = HDP == 32 ? 2 : 1;
  constexpr int P_OFF = NST * STAGE_BYTES;
  constexpr int DS_OFF = P_OFF + AT_ROWS * 128 * 2;
  constexpr int ACC_OFF = DS_OFF + AT_ROWS * 128 * 2;
  constexpr int BIAS_OFF = ACC_OFF + AT_ACC_BYTES;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int S = p.S;
  const int SS = (S * S * 4 + 15) & ~15;
  float* bias_s = reinterpret_cast<float*>(smem + BIAS_OFF);
  float* acc = reinterpret_cast<float*>(smem + ACC_OFF);
  uint8_t* ctrl = smem + BIAS_OFF + SS;
  uint64_t* ld_full = reinterpret_cast<uint64_t*>(ctrl);  // [2]
  uint64_t* ld_empty = ld_full + 2;                        // [2]

  if (warp == AT_PRODUCER && lane == 0) {
    tma_prefetch_desc(&tmap_qkv);
    tma_prefetch_desc(&tmap_do);
    if (HT::HB > 0) tma_prefetch_desc(&tmap_qkv_b), tma_prefetch_desc(&tmap_do_b);
    for (int i = 0; i < 2; ++i) {
      mbar_init(&ld_full[i], 1);
      mbar_init(&ld_empty[i], 1);
    }
    fence_mbar_init();
  }
  __syncthreads();

  const int nslots = AT_ROWS / p.slot;
  // Item order: with at least one CTA per head every CTA stays on ONE head (CTA c: head c % heads, every n_h-th tile
  // of it), so a thread's share of dbias[head] -- row j of its window slot -- accumulates in registers over all of
  // the CTA's items and is flushed with one global atomic per element at the end. Smaller grids walk head-major.
  const bool by_head = (int)gridDim.x >= p.heads;
  const int my_head = by_head ? (int)blockIdx.x % p.heads : 0;
  const int n_h = by_head ? ((int)gridDim.x - my_head + p.heads - 1) / p.heads : 1;
  const int q_h = (int)blockIdx.x / p.heads;
  const int n_items = by_head ? (q_h < p.tiles ? (p.tiles - q_h + n_h - 1) / n_h : 0)
                              : (p.tiles * p.heads - (int)blockIdx.x + (int)gridDim.x - 1) / (int)gridDim.x;
  auto item_of = [&](int it, int& head, int& tile) {
    if (by_head) {
      head = my_head, tile = q_h + it * n_h;
    } else {
      const int w = (int)blockIdx.x + it * (int)gridDim.x;
      head = w / p.tiles, tile = w % p.tiles;
    }
  };

  if (warp == AT_PRODUCER) {
    if (lane == 0) {
      for (int it = 0; it < n_items; ++it) {
        const int st = it % NST;
        const uint32_t ph = (it / NST) & 1;
        int head, tile;
        item_of(it, head, tile);
        mbar_wait(&ld_empty[st], ph ^ 1);
        uint8_t* base = smem + st * STAGE_BYTES;
        mbar_expect_tx(&ld_full[st], STAGE_BYTES);
        for (int sl = 0; sl < nslots; ++sl) {
          const int row0 = (tile * p.gpt + sl) * S;
          for (int op = 0; op < 3; ++op)
            HT::load(base + op * TILE_BYTES, AT_ROWS, sl * p.slot, &tmap_qkv, &tmap_qkv_b, &ld_full[st],
                     (op * p.heads + head) * HDP, row0);
          HT::load(base + 3 * TILE_BYTES, AT_ROWS, sl * p.slot, &tmap_do, &tmap_do_b, &ld_full[st], head * HDP, row0);
        }
      }
    }
  } else {
    const int quad = warp & 3;
    const int r = quad * 32 + lane;
    const int tid = threadIdx.x;
    const float* arow = acc + r * AT_ACC_LD;
    const int slot = p.slot;
    const int sl = r / slot;
    const int j = r - sl * slot;
    const int lo = sl * slot;
    const int wlo = slot >= 32 ? lo : quad * 32;
    const int wn = slot >= 32 ? S : 32;
    const int nch = (wn + 31) / 32;  // <= 2 (S <= 64)
    uint8_t* sP = smem + P_OFF;
    uint8_t* sDS = smem + DS_OFF;
    for (int c = 0; c < 128; c += 8) {
      if (c + 8 <= wlo || c >= wlo + 32 * nch) {
        const uint32_t off = (c >> 6) * (AT_ROWS * 128) + r * 128 + ((((c & 63) >> 3) ^ (r & 7)) << 4);
        *reinterpret_cast<uint4*>(sP + off) = make_uint4(0, 0, 0, 0);
        *reinterpret_cast<uint4*>(sDS + off) = make_uint4(0, 0, 0, 0);
      }
    }
    int staged_head = -1;
    float dacc[64];  // this thread's share of dbias[head]: row j, the 64 key columns of its chunks
#pragma unroll
    for (int u = 0; u < 64; ++u) dacc[u] = 0.f;
    auto flush_dbias = [&](int head) {
      if (p.dbias == nullptr || head < 0) return;
      if (j < S && sl < p.gpt) {
        float* dst = p.dbias + ((long long)head * S + j) * S;
#pragma unroll
        for (int u = 0; u < 64; ++u) {
          const int kk = wlo + u - lo;
          if (u < 32 * nch && kk >= 0 && kk < S && dacc[u] != 0.f) atomicAdd(dst + kk, dacc[u]);
        }
      }
#pragma unroll
      for (int u = 0; u < 64; ++u) dacc[u] = 0.f;
    };
    for (int it = 0; it < n_items; ++it) {
      int head, tile;
      item_of(it, head, tile);
      const int grp = tile * p.gpt + sl;
      const bool row_ok = j < S && sl < p.gpt && grp < p.groups;
      if (head != staged_head) {
        flush_dbias(staged_head);
        named_bar_sync(1, 128);
        if (p.bias) {
          const float* bsrc = p.bias + (long long)head * S * S;
          const int n = S * S;
          for (int i0 = tid; i0 < n; i0 += 128 * 8) {
            float tmp[8];
#pragma unroll
            for (int u = 0; u < 8; ++u) {
              const int i = i0 + u * 128;
              tmp[u] = i < n ? __ldg(bsrc + i) : 0.f;
            }
#pragma unroll
            for (int u = 0; u < 8; ++u) {
              const int i = i0 + u * 128;
              if (i < n) bias_s[i] = tmp[u] * 1.4426950408889634f;
            }
          }
        }
        named_bar_sync(1, 128);
        staged_head = head;
      }
      const int st = it % NST;
      mbar_wait(&ld_full[st], (it / NST) & 1);
      const uint32_t sQ = smem_u32(smem + st * STAGE_BYTES);
      const uint32_t sK = sQ + TILE_BYTES, sV = sQ + 2 * TILE_BYTES, sDO = sQ + 3 * TILE_BYTES;
      const uint32_t sPu = smem_u32(sP), sDSu = smem_u32(sDS);
      named_bar_sync(1, 128);  // the previous item's gradient reads of the accumulator tile are done
      wg_mma_128<128, 0, 0, HT::KSTEPS>(
          acc, AT_ACC_LD, [&](int h, int k) { return HT::kdesc(sQ, AT_ROWS, h * 64, k); },
          [&](int k) { return HT::kdesc(sK, AT_ROWS, 0, k); }, false);
      named_bar_sync(1, 128);
      const float* brow = bias_s + (row_ok ? j : 0) * S;
      const bool use_bias = p.bias != nullptr;
      float e[64];
      float mx = -INFINITY;
#pragma unroll
      for (int ch = 0; ch < 2; ++ch) {
        if (ch < nch) {
          const int c0 = wlo + 32 * ch;
          uint32_t raw[32];
          ld_row32(arow + c0, raw);
#pragma unroll
          for (int u = 0; u < 32; ++u) {
            const int kk = c0 + u - lo;
            const bool in = kk >= 0 && kk < S;
            const float b = use_bias ? brow[in ? kk : 0] : 0.f;
            const float sc = in ? fmaf(__uint_as_float(raw[u]), p.scale_log2e, b) : -INFINITY;
            e[32 * ch + u] = sc;
            mx = fmaxf(mx, sc);
          }
        } else {
#pragma unroll
          for (int u = 0; u < 32; ++u) e[32 * ch + u] = -INFINITY;
        }
      }
      if (!row_ok) mx = 0.f;
      float sum = 0.f;
#pragma unroll
      for (int u = 0; u < 64; ++u) {
        const float v = row_ok ? exp2f(e[u] - mx) : 0.f;  // exp2(-inf) = 0 outside the window
        e[u] = v;
        sum += v;
      }
      const float inv = row_ok ? 1.f / sum : 0.f;
      named_bar_sync(1, 128);  // every score read is done: dP = dO V^T overwrites the tile
      wg_mma_128<128, 0, 0, HT::KSTEPS>(
          acc, AT_ACC_LD, [&](int h, int k) { return HT::kdesc(sDO, AT_ROWS, h * 64, k); },
          [&](int k) { return HT::kdesc(sV, AT_ROWS, 0, k); }, false);
      named_bar_sync(1, 128);
      float delta = 0.f;
#pragma unroll
      for (int ch = 0; ch < 2; ++ch) {
        if (ch < nch) {
          const int c0 = wlo + 32 * ch;
          uint32_t raw[32];
          ld_row32(arow + c0, raw);
#pragma unroll
          for (int u = 0; u < 32; ++u) {
            e[32 * ch + u] *= inv;  // normalised probability
            delta = fmaf(e[32 * ch + u], __uint_as_float(raw[u]), delta);
          }
        }
      }
#pragma unroll
      for (int ch = 0; ch < 2; ++ch) {
        if (ch < nch) {
          const int c0 = wlo + 32 * ch;
          uint32_t raw[32];
          ld_row32(arow + c0, raw);
          uint32_t pkp[16], pkd[16];
#pragma unroll
          for (int u = 0; u < 32; u += 2) {
            float ds[2];
#pragma unroll
            for (int t = 0; t < 2; ++t) {
              const float pv = e[32 * ch + u + t];
              ds[t] = pv * (__uint_as_float(raw[u + t]) - delta);
              dacc[32 * ch + u + t] += ds[t];   // (pv = 0 outside the window / for rows that are not real queries)
            }
            const __half2 hp = __floats2half2_rn(e[32 * ch + u], e[32 * ch + u + 1]);
            const __half2 hd = __floats2half2_rn(ds[0], ds[1]);
            pkp[u >> 1] = *reinterpret_cast<const uint32_t*>(&hp);
            pkd[u >> 1] = *reinterpret_cast<const uint32_t*>(&hd);
          }
#pragma unroll
          for (int q = 0; q < 4; ++q) {
            const int c = c0 + q * 8;
            if (c < 128) {
              const uint32_t off = (c >> 6) * (AT_ROWS * 128) + r * 128 + ((((c & 63) >> 3) ^ (r & 7)) << 4);
              *reinterpret_cast<uint4*>(sP + off) = make_uint4(pkp[4 * q], pkp[4 * q + 1], pkp[4 * q + 2], pkp[4 * q + 3]);
              *reinterpret_cast<uint4*>(sDS + off) = make_uint4(pkd[4 * q], pkd[4 * q + 1], pkd[4 * q + 2], pkd[4 * q + 3]);
            }
          }
        }
      }
      fence_proxy_async_smem();
      // gradients: row r of dV / dK is key r, of dQ is query r — the same token of the window
      const long long grow = (long long)grp * S + j;
      __half* orow = p.dqkv + grow * p.lddq + head * HDP;
      const int Cp = p.heads * HDP;
#pragma unroll 1
      for (int which = 0; which < 3; ++which) {
        named_bar_sync(1, 128);  // P / dS are complete, the previous tile reads are done
        if (which == 0) {        // dQ = dS K
          wg_mma_128_head<HDP, 0, 8>(
              acc, AT_ACC_LD,
              [&](int h, int ks) {
                return make_smem_desc(sDSu + (ks >> 2) * (AT_ROWS * 128) + h * 64 * 128 + (ks & 3) * 32, 16, 1024, SWZ_128B);
              },
              sK, AT_ROWS, false);
        } else {                 // dK = dS^T Q, dV = P^T dO: A read MN-major (M = keys), K = 128 query rows
          const uint32_t sA = which == 1 ? sDSu : sPu;
          const uint32_t sB = which == 1 ? sQ : sDO;
          wg_mma_128_head<HDP, 1, 8>(
              acc, AT_ACC_LD,
              [&](int h, int ks) { return make_smem_desc(sA + h * (AT_ROWS * 128) + ks * 2048, AT_ROWS * 128, 1024, SWZ_128B); },
              sB, AT_ROWS, false);
        }
        named_bar_sync(1, 128);
        if (which == 2 && tid == 0) mbar_arrive(&ld_empty[st]);  // Q / K / V / dO of this stage are consumed
        const float mul = which == 2 ? 1.f : p.scale;
        if (row_ok) store_row_f16<HDP>(arow, mul, orow + which * Cp);
      }
    }
    flush_dbias(staged_head);
  }
}

template <int HDP>
static int launch_attn_bwd(const CUtensorMap& tq, const CUtensorMap& td, const CUtensorMap& tqb, const CUtensorMap& tdb,
                           const AttnBwdParams& p, size_t smem, cudaStream_t st) {
  static bool configured = false;
  if (!configured) {
    FVIT_CUDA(cudaFuncSetAttribute(attn_bwd_tc_kernel<HDP>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
    configured = true;
  }
  const int items = p.tiles * p.heads;
  const int sms = num_sms();
  attn_bwd_tc_kernel<HDP><<<items < sms ? items : sms, AT_THREADS, smem, st>>>(tq, td, tqb, tdb, p);
  return post_launch("attn_bwd_tc_kernel");
}

}  // namespace fvit

extern "C" int fvit_attn_tc_bwd(const void* qkv, int64_t ldq, const void* dout, int64_t lddo, int32_t groups, int32_t S,
                                int32_t heads, int32_t head_dim, int32_t hdp, const float* bias, float scale, void* dqkv,
                                int64_t lddq, float* dbias, void* stream) {
  using namespace fvit;
  FVIT_CHECK(qkv && dout && dqkv && groups > 0 && heads > 0, "fvit_attn_tc_bwd: bad arguments");
  FVIT_CHECK(S >= 1 && S <= 64, "fvit_attn_tc_bwd: S=%d unsupported (1..64)", S);
  FVIT_CHECK(hdp == 32 || hdp == 64 || hdp == 80, "fvit_attn_tc_bwd: padded head dim %d unsupported", hdp);
  FVIT_CHECK(ldq % 8 == 0 && lddo % 8 == 0 && lddq % 8 == 0, "fvit_attn_tc_bwd: bad leading dimensions");
  AttnBwdParams p;
  p.groups = groups, p.S = S, p.heads = heads, p.hd = head_dim;
  p.slot = S <= 16 ? 16 : (S <= 32 ? 32 : 64);
  p.gpt = AT_ROWS / p.slot;
  p.tiles = (groups + p.gpt - 1) / p.gpt;
  p.scale = scale;
  p.scale_log2e = scale * 1.4426950408889634f;
  p.bias = bias, p.dbias = dbias;
  p.dqkv = (__half*)dqkv, p.lddq = lddq;
  const int rows_total = groups * S;
  CUtensorMap tq, td, tqb, tdb;
  int rc = head_tile_tmaps(&tq, &tqb, qkv, 3 * heads * hdp, rows_total, ldq, hdp, p.slot);
  if (rc) return rc;
  rc = head_tile_tmaps(&td, &tdb, dout, heads * hdp, rows_total, lddo, hdp, p.slot);
  if (rc) return rc;
  const size_t ss = ((size_t)S * S * 4 + 15) / 16 * 16;
  const size_t smem = 1024 + (size_t)(hdp == 32 ? 2 : 1) * 4 * AT_ROWS * hdp * 2 + 2 * AT_ROWS * 128 * 2 + AT_ACC_BYTES + ss + 128;
  FVIT_CHECK(smem <= 227 * 1024, "fvit_attn_tc_bwd: needs %zu B of shared memory", smem);
  if (hdp == 80) return launch_attn_bwd<80>(tq, td, tqb, tdb, p, smem, (cudaStream_t)stream);
  if (hdp == 64) return launch_attn_bwd<64>(tq, td, tqb, tdb, p, smem, (cudaStream_t)stream);
  return launch_attn_bwd<32>(tq, td, tqb, tdb, p, smem, (cudaStream_t)stream);
}
