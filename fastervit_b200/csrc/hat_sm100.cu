// fvit_hat_attn_fwd: the fused hierarchical-attention kernel of WindowAttention.forward (fv.py:557-565) for sm_90a —
// QKV projection, softmax(Q K^T * scale + relative-position bias) and the V contraction in ONE wgmma kernel; the
// [tokens, 3C] qkv matrix and the score / probability matrices never exist in HBM (inference), or qkv is written once
// and never read back (training, where the backward pass needs it).
//
// Work item = (tile of 128 token rows = gpt whole windows in slots of 16/32/64/128 rows, head); head-major order so the
// head's weight slice [3*hdp, C] and bias [S, S] stay hot in L2 / shared memory.
//
//   warp 4     : TMA producer — per 64-wide K block the (window_size^2 + ct_size^2) x 64 activation boxes of the tile's
//                windows and the head's W_q / W_k / W_v boxes into a ring of 128B-swizzled stages
//   warps 0..3 : one warpgroup — (1) [Q | K | V] = X W_h^T over C (wgmma, register accumulators) + qkv bias -> fp16
//                straight from the accumulator fragments into the swizzled Q / K / V operand tiles (and optionally the
//                qkv matrix for the backward pass); (2) S = Q K^T into an fp32 score tile, softmax with one thread per
//                token row (block-diagonal mask, bias from shared memory, exp2), P as fp16 operand; (3) O = P V into the
//                score tile, O / rowsum -> fp16 out.
// The score tile shares its shared memory with the operand ring: the producer starts an item's loads once the previous
// item's O has been read out (ring_free).
#include <cuda_fp16.h>

#include "../../include/fvit.h"
#include "common.h"
#include "ptx.cuh"

namespace fvit {

constexpr int HT_THREADS = 160;
constexpr int HT_ROWS = 128;
constexpr int HT_BK = 64;
constexpr int HT_MAX_STAGES = 4;
constexpr int HT_PRODUCER = 4;   // the TMA warp; warps 0..3 are the compute warpgroup
constexpr int HT_ACC_LD = 132;   // floats per row of the fp32 score tile
constexpr int HT_ACC_BYTES = HT_ROWS * HT_ACC_LD * 4;

struct HatParams {
  int groups, S, heads, gpt, tiles, slot;
  int num_kb;   // ceil(C / 64)
  int k_tail16; // 16-wide MMA steps with real columns in the last K-block (the rest is TMA zero fill: not issued)
  int stages;
  int ring_bytes;  // operand ring / score tile region
  int Cp;       // heads * hdp
  float scale_log2e;
  const float* qkv_bias;  // [3 * Cp] head-padded, or null
  const float* bias;      // [heads, S, S] or null
  __half* out;
  long long ldo;
  __half* qkv_out;        // optional [rows, 3 * Cp]
  long long ldq;
  int rows_total;
};

template <int HDP>
__global__ void __launch_bounds__(HT_THREADS, 1)
    hat_attn_kernel(const __grid_constant__ CUtensorMap tmap_x, const __grid_constant__ CUtensorMap tmap_w,
                    const __grid_constant__ HatParams p) {
  static_assert(HDP == 64, "the Q / K / V operand tiles are 128-byte rows in the 128B swizzle");
  constexpr uint32_t ROW_BYTES = HDP * 2;
  constexpr uint32_t SBO_QKV = 8 * ROW_BYTES;
  constexpr int A_BYTES = HT_ROWS * HT_BK * 2;        // 16 KB
  constexpr int B_BYTES = 3 * HDP * HT_BK * 2;        // 24 KB
  constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
  constexpr int OPER_BYTES = HT_ROWS * HDP * 2;       // one of Q / K / V as fp16 operand tile
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int S = p.S;
  float* sacc = reinterpret_cast<float*>(smem);             // score / O tile, aliases the operand ring
  uint8_t* s_oper = smem + p.ring_bytes;                    // Q, K, V operand tiles
  uint8_t* s_p = s_oper + 3 * OPER_BYTES;                   // P: 128 x 128 fp16 (two 64-wide K atoms)
  float* bias_s = reinterpret_cast<float*>(s_p + HT_ROWS * 128 * 2);
  uint8_t* ctrl = reinterpret_cast<uint8_t*>(bias_s) + ((S * S * 4 + 15) & ~15);
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(ctrl);   // [HT_MAX_STAGES]
  uint64_t* empty_bar = full_bar + HT_MAX_STAGES;           // [HT_MAX_STAGES]
  uint64_t* ring_free = empty_bar + HT_MAX_STAGES;

  if (warp == HT_PRODUCER && lane == 0) {
    tma_prefetch_desc(&tmap_x);
    tma_prefetch_desc(&tmap_w);
    for (int i = 0; i < p.stages; ++i) mbar_init(&full_bar[i], 1), mbar_init(&empty_bar[i], 4);
    mbar_init(ring_free, 1);
    fence_mbar_init();
  }
  __syncthreads();

  const int items = p.tiles * p.heads;
  const int nslots = HT_ROWS / p.slot;

  if (warp == HT_PRODUCER) {
    // ===================================================================== TMA producer
    if (lane == 0) {
      int stage = 0;
      uint32_t phase = 0, it = 0;
      for (int w = blockIdx.x; w < items; w += gridDim.x, ++it) {
        const int head = w / p.tiles, tile = w % p.tiles;
        mbar_wait(ring_free, (it & 1) ^ 1);  // the previous item's score tile has been read out
        for (int kb = 0; kb < p.num_kb; ++kb) {
          mbar_wait(&empty_bar[stage], phase ^ 1);
          uint8_t* sa = smem + stage * STAGE_BYTES;
          uint8_t* sb = sa + A_BYTES;
          mbar_expect_tx(&full_bar[stage], STAGE_BYTES);
          for (int sl = 0; sl < nslots; ++sl)  // window (tile*gpt + sl) -> rows [sl*slot, (sl+1)*slot); OOB rows are zero
            tma_load_2d(sa + sl * p.slot * 128, &tmap_x, &full_bar[stage], kb * HT_BK, (tile * p.gpt + sl) * S);
#pragma unroll
          for (int which = 0; which < 3; ++which)
            tma_load_2d(sb + which * (HDP * 128), &tmap_w, &full_bar[stage], kb * HT_BK, which * p.Cp + head * HDP);
          if (++stage == p.stages) stage = 0, phase ^= 1;
        }
      }
    }
  } else {
    // ===================================================================== compute warpgroup
    const int quad = warp & 3;
    const int r = quad * 32 + lane;    // row in tile
    const int tid = threadIdx.x;       // 0..127
    const int slot = p.slot;
    const int sl = r / slot;
    const int j = r - sl * slot;       // token index inside the window
    const int lo = sl * slot;
    const int wlo = slot >= 32 ? lo : quad * 32;
    const int wn = slot >= 32 ? S : 32;
    const int nch = (wn + 31) / 32;
    const float* arow = sacc + r * HT_ACC_LD;
    const uint32_t sQ = smem_u32(s_oper), sK = sQ + OPER_BYTES, sV = sK + OPER_BYTES, sPu = smem_u32(s_p);
    // columns of P outside the warp's windows are never written: zero them once
    for (int c = 0; c < 128; c += 8) {
      if (c + 8 <= wlo || c >= wlo + 32 * nch)
        *reinterpret_cast<uint4*>(s_p + (c >> 6) * (HT_ROWS * 128) + r * 128 + ((((c & 63) >> 3) ^ (r & 7)) << 4)) =
            make_uint4(0, 0, 0, 0);
    }
    // byte offset of element (row, col) inside a Q / K / V operand tile (128B swizzle)
    auto oper_off = [&](int row, int col) -> uint32_t {
      return (uint32_t)(row * 128 + ((((col >> 3) ^ (row & 7))) << 4) + (col & 7) * 2);
    };
    int stage = 0;
    uint32_t phase = 0, it = 0;
    int staged_head = -1;
    for (int w = blockIdx.x; w < items; w += gridDim.x, ++it) {
      const int head = w / p.tiles, tile = w % p.tiles;
      const int grp = tile * p.gpt + sl;
      const bool row_ok = j < S && sl < p.gpt && grp < p.groups;
      const long long grow = (long long)grp * S + j;
      if (p.bias && head != staged_head) {
        named_bar_sync(1, 128);
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
      // ---- (1) projection: [Q | K | V] rows 64h .. 64h + 63 in registers, K blocks from the ring
      {
        float d[2][3][HDP / 2];
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
          for (int which = 0; which < 3; ++which)
#pragma unroll
            for (int u = 0; u < HDP / 2; ++u) d[h][which][u] = 0.f;
        for (int kb = 0; kb < p.num_kb; ++kb) {
          mbar_wait(&full_bar[stage], phase);
          const uint32_t sa = smem_u32(smem + stage * STAGE_BYTES), sb = sa + A_BYTES;
          const int nk = kb + 1 == p.num_kb ? p.k_tail16 : HT_BK / 16;
          auto step = [&](int k) {
#pragma unroll
            for (int h = 0; h < 2; ++h)
#pragma unroll
              for (int which = 0; which < 3; ++which)
                Wgmma<HDP, 0, 0, 0>::mma(d[h][which], make_smem_desc(sa + h * 8192 + k * 32, 16, 1024, SWZ_128B),
                                         make_smem_desc(sb + which * (HDP * 128) + k * 32, 16, 1024, SWZ_128B), 1u);
          };
          // (each case is a complete wgmma group: a branch between the MMAs of one group would serialize them)
          switch (nk) {
            case 1: wgmma_fence(); step(0); wgmma_commit(); break;
            case 2: wgmma_fence(); step(0); step(1); wgmma_commit(); break;
            case 3: wgmma_fence(); step(0); step(1); step(2); wgmma_commit(); break;
            default: wgmma_fence(); step(0); step(1); step(2); step(3); wgmma_commit(); break;
          }
          wgmma_wait0();
          __syncwarp();
          if (lane == 0) mbar_arrive(&empty_bar[stage]);
          if (++stage == p.stages) stage = 0, phase ^= 1;
        }
        // accumulator fragments (+ qkv bias) -> fp16 operand tiles (+ optional global copy of the qkv rows)
        const int t = tid & 127;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
#pragma unroll
          for (int half8 = 0; half8 < 2; ++half8) {
            const int row = h * 64 + (t >> 5) * 16 + ((t & 31) >> 2) + half8 * 8;
            const int rsl = row / slot, rj = row - rsl * slot, rgrp = tile * p.gpt + rsl;
            const bool rok = rj < S && rsl < p.gpt && rgrp < p.groups;
            __half* gq = (p.qkv_out && rok) ? p.qkv_out + ((long long)rgrp * S + rj) * p.ldq + head * HDP : nullptr;
#pragma unroll
            for (int which = 0; which < 3; ++which) {
              const float* qb = p.qkv_bias ? p.qkv_bias + which * p.Cp + head * HDP : nullptr;
              uint8_t* dst = s_oper + which * OPER_BYTES;
#pragma unroll
              for (int jj = 0; jj < HDP / 8; ++jj) {
                const int col = jj * 8 + 2 * (t & 3);
                const float b0 = qb ? __ldg(qb + col) : 0.f, b1 = qb ? __ldg(qb + col + 1) : 0.f;
                const __half2 hh = __floats2half2_rn(d[h][which][4 * jj + 2 * half8] + b0, d[h][which][4 * jj + 2 * half8 + 1] + b1);
                *reinterpret_cast<__half2*>(dst + oper_off(row, col)) = hh;
                if (gq) *reinterpret_cast<__half2*>(gq + which * p.Cp + col) = hh;
              }
            }
          }
        }
      }
      fence_proxy_async_smem();
      named_bar_sync(1, 128);  // Q / K / V complete; the previous item's O reads are done
      // ---- (2) scores and softmax over the window's keys
      wg_mma_128<128, 0, 0, HDP / 16>(
          sacc, HT_ACC_LD,
          [&](int h, int k) { return make_smem_desc(sQ + h * 64 * ROW_BYTES + k * 32, 16, SBO_QKV, SWZ_128B); },
          [&](int k) { return make_smem_desc(sK + k * 32, 16, SBO_QKV, SWZ_128B); }, false);
      named_bar_sync(1, 128);
      const float* brow = bias_s + (row_ok ? j : 0) * S;
      const bool use_bias = p.bias != nullptr;
      float mx = -INFINITY;
      for (int ch = 0; ch < nch; ++ch) {
        const int c0 = wlo + 32 * ch;
        uint32_t raw[32];
        ld_row32(arow + c0, raw);
#pragma unroll
        for (int u = 0; u < 32; ++u) {
          const int kk = c0 + u - lo;
          const bool in = kk >= 0 && kk < S;
          const float b = use_bias ? brow[in ? kk : 0] : 0.f;
          const float sc = fmaf(__uint_as_float(raw[u]), p.scale_log2e, b);
          mx = fmaxf(mx, in ? sc : -INFINITY);
        }
      }
      if (!row_ok) mx = 0.f;
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
          sum += __low2float(h) + __high2float(h);
          pk[u >> 1] = *reinterpret_cast<const uint32_t*>(&h);
        }
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const int c = c0 + q * 8;
          if (c < 128)
            *reinterpret_cast<uint4*>(s_p + (c >> 6) * (HT_ROWS * 128) + r * 128 + ((((c & 63) >> 3) ^ (r & 7)) << 4)) =
                make_uint4(pk[4 * q], pk[4 * q + 1], pk[4 * q + 2], pk[4 * q + 3]);
        }
      }
      fence_proxy_async_smem();
      named_bar_sync(1, 128);  // P complete, score reads done
      // ---- (3) O = P V, epilogue
      wg_mma_128<HDP, 0, 1, 8>(
          sacc, HT_ACC_LD,  // 128 keys in steps of 16
          [&](int h, int ks) {
            return make_smem_desc(sPu + (ks >> 2) * (HT_ROWS * 128) + h * 64 * 128 + (ks & 3) * 32, 16, 1024, SWZ_128B);
          },
          [&](int ks) { return make_smem_desc(sV + ks * 16 * ROW_BYTES, 0, SBO_QKV, SWZ_128B); }, false);
      named_bar_sync(1, 128);
      const float inv = row_ok ? 1.f / sum : 0.f;
      __half* orow = p.out + grow * p.ldo + head * HDP;
#pragma unroll
      for (int c0 = 0; c0 < HDP; c0 += 32) {
        uint32_t raw[32];
        ld_row32(arow + c0, raw);
        if (row_ok) {
#pragma unroll
          for (int q = 0; q < 4; ++q) {
            uint32_t o4[4];
#pragma unroll
            for (int u = 0; u < 4; ++u) {
              const __half2 h = __floats2half2_rn(__uint_as_float(raw[q * 8 + 2 * u]) * inv,
                                                  __uint_as_float(raw[q * 8 + 2 * u + 1]) * inv);
              o4[u] = *reinterpret_cast<const uint32_t*>(&h);
            }
            *reinterpret_cast<uint4*>(orow + c0 + q * 8) = make_uint4(o4[0], o4[1], o4[2], o4[3]);
          }
        }
      }
      named_bar_sync(1, 128);
      if (tid == 0) mbar_arrive(ring_free);  // the score tile is read out: the ring may take the next item's loads
    }
  }
}

template <int HDP>
static int launch_hat(const CUtensorMap& tx, const CUtensorMap& tw, HatParams& p, cudaStream_t st) {
  constexpr int STAGE_BYTES = HT_ROWS * HT_BK * 2 + 3 * HDP * HT_BK * 2;
  const size_t fixed = 1024 + (size_t)3 * HT_ROWS * HDP * 2 + HT_ROWS * 128 * 2 + (((size_t)p.S * p.S * 4 + 15) & ~(size_t)15) + 256;
  int stages = (int)((227 * 1024 - fixed) / STAGE_BYTES);
  if (stages > HT_MAX_STAGES) stages = HT_MAX_STAGES;
  FVIT_CHECK(stages >= 2, "fvit_hat_attn_fwd: S=%d leaves no room for a 2-stage operand ring", p.S);
  p.stages = stages;
  p.ring_bytes = stages * STAGE_BYTES > HT_ACC_BYTES ? stages * STAGE_BYTES : HT_ACC_BYTES;
  const size_t smem = fixed + (size_t)p.ring_bytes;
  FVIT_CHECK(smem <= 227 * 1024, "fvit_hat_attn_fwd: S=%d needs %zu B of shared memory", p.S, smem);
  static bool configured = false;
  if (!configured) {
    FVIT_CUDA(cudaFuncSetAttribute(hat_attn_kernel<HDP>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
    configured = true;
  }
  const int items = p.tiles * p.heads;
  const int sms = num_sms();
  hat_attn_kernel<HDP><<<items < sms ? items : sms, HT_THREADS, smem, st>>>(tx, tw, p);
  return post_launch("hat_attn_kernel");
}

}  // namespace fvit

using namespace fvit;

extern "C" int fvit_hat_attn_fwd(const void* xn16, int64_t ldx, int32_t C, const void* wqkv16, int64_t ldw,
                                 const float* qkv_bias, int32_t groups, int32_t S, int32_t heads, int32_t hdp,
                                 const float* bias, float scale, void* out, int64_t ldo, void* qkv_out, int64_t ldq,
                                 void* stream) {
  FVIT_CHECK(xn16 && wqkv16 && out && groups > 0 && heads > 0 && C > 0, "fvit_hat_attn_fwd: bad arguments");
  FVIT_CHECK(S >= 1 && S <= 128, "fvit_hat_attn_fwd: S=%d unsupported (1..128)", S);
  FVIT_CHECK(hdp == 64, "fvit_hat_attn_fwd: padded head dim %d unsupported (64 only)", hdp);
  FVIT_CHECK(ldx % 8 == 0 && ldw % 8 == 0 && ldo % 8 == 0 && ldo >= heads * hdp, "fvit_hat_attn_fwd: bad leading dimensions");
  FVIT_CHECK(!qkv_out || (ldq % 8 == 0 && ldq >= 3 * heads * hdp), "fvit_hat_attn_fwd: bad qkv_out leading dimension");
  FVIT_CHECK((reinterpret_cast<uintptr_t>(out) & 15) == 0 && (reinterpret_cast<uintptr_t>(qkv_out) & 15) == 0,
             "fvit_hat_attn_fwd: outputs must be 16-byte aligned");
  HatParams p;
  memset(&p, 0, sizeof(p));
  p.groups = groups, p.S = S, p.heads = heads;
  p.slot = S <= 16 ? 16 : (S <= 32 ? 32 : (S <= 64 ? 64 : 128));
  p.gpt = HT_ROWS / p.slot;
  p.tiles = (groups + p.gpt - 1) / p.gpt;
  p.num_kb = (C + HT_BK - 1) / HT_BK;
  p.k_tail16 = (C - (p.num_kb - 1) * HT_BK + 15) / 16;
  p.Cp = heads * hdp;
  p.scale_log2e = scale * 1.4426950408889634f;
  p.qkv_bias = qkv_bias, p.bias = bias;
  p.out = (__half*)out, p.ldo = ldo, p.qkv_out = (__half*)qkv_out, p.ldq = ldq;
  p.rows_total = groups * S;
  CUtensorMap tx, tw;
  {
    uint64_t dims[2] = {(uint64_t)C, (uint64_t)p.rows_total};
    uint64_t strides[1] = {(uint64_t)ldx * 2};
    uint32_t box[2] = {(uint32_t)HT_BK, (uint32_t)p.slot};
    int rc = cached_tmap_16bit(&tx, xn16, 2, dims, strides, box, CU_TENSOR_MAP_SWIZZLE_128B);
    if (rc) return rc;
    uint64_t dimsw[2] = {(uint64_t)C, (uint64_t)(3 * p.Cp)};
    uint64_t stridesw[1] = {(uint64_t)ldw * 2};
    uint32_t boxw[2] = {(uint32_t)HT_BK, (uint32_t)hdp};
    rc = cached_tmap_16bit(&tw, wqkv16, 2, dimsw, stridesw, boxw, CU_TENSOR_MAP_SWIZZLE_128B);
    if (rc) return rc;
  }
  return launch_hat<64>(tx, tw, p, (cudaStream_t)stream);
}
