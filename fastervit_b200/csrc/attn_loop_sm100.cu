// fvit_attn_loop_fwd: tensor-core attention core of WindowAttention.forward (fv.py:559-565; fvar.py:805-817 for the
// any-res level-2 geometry S = 12*12 + 4 = 148; fv.py:1253-1418 for the 21k windows S = 196 .. 2304) for window
// sequences longer than one 128-row tile.
//
// Work item = (window, head, tile of 128 query rows). Keys are visited in tiles of 128, twice:
//   pass 1: S_j = Q K_j^T (wgmma, 128 x 128 fp32 in a shared-memory tile) -> running row maximum of S_j*scale + bias
//   pass 2: S_j again, P_j = exp2(S_j*scale*log2e + bias*log2e - max) as fp16 into the swizzled operand tile,
//           O += P_j V_j (fp32 shared-memory accumulator over the key tiles), row sums of the rounded probabilities
// so no accumulator is ever rescaled; the score recomputation is 2*S*S*hd FLOPs of a contraction that is < 3 % of
// the model. Scores / probabilities never touch HBM.
//
//   warp 4     : TMA producer  — Q tile, K / V tiles through a 2-stage ring (1 at hdp 80), relative-position-bias tiles
//                (fp32 [128 rows x 32 keys] units, one 128B-swizzled box each) through a 2-stage ring, all in the
//                order the compute warpgroup consumes them
//   warps 0..3 : one warpgroup — the score and P V MMAs (wgmma, two m64 halves), softmax with one thread per query
//                row (bias from shared memory, exp2, P store), then the O epilogue (1 / rowsum, fp16, 16-byte
//                stores) and the optional log-sum-exp row vector
#include <cuda_fp16.h>

#include "../../include/fvit.h"
#include "attn_head.cuh"
#include "common.h"
#include "ptx.cuh"

namespace fvit {

constexpr int AL_THREADS = 160;
constexpr int AL_ROWS = 128;
constexpr int AL_PRODUCER = 4;  // the TMA warp; warps 0..3 are the compute warpgroup
constexpr int AL_NB = 2;        // bias unit ring depth
constexpr int AL_BUNIT = 32;    // key columns per bias unit
constexpr int AL_ACC_LD = 132;  // floats per row of the fp32 score tile


struct AttnLoopParams {
  int groups, S, heads, nqt, nkt;
  float scale_log2e;
  int has_bias;
  __half* out;
  long long ldo;
  float* lse;  // optional [groups * S, heads]: log2-domain log-sum-exp of the scaled, biased scores
};

template <int HDP>
struct AttnLoopSmem {
  static constexpr int TILE_BYTES = AL_ROWS * HDP * 2;
  // K / V tile ring depth: at HDP 80 a second stage would push the layout past 227 KB
  static constexpr int NKV = HDP == 80 ? 1 : 2;
  static constexpr int BUNIT_BYTES = AL_ROWS * AL_BUNIT * 4;
  static constexpr int O_LD = HDP + 4;
  static constexpr int Q_OFF = 0;
  static constexpr int KV_OFF = TILE_BYTES;
  static constexpr int P_OFF = KV_OFF + NKV * TILE_BYTES;
  static constexpr int BIAS_OFF = P_OFF + AL_ROWS * 128 * 2;
  static constexpr int SACC_OFF = BIAS_OFF + AL_NB * BUNIT_BYTES;
  static constexpr int OACC_OFF = SACC_OFF + AL_ROWS * AL_ACC_LD * 4;
  static constexpr int CTRL_OFF = OACC_OFF + AL_ROWS * O_LD * 4;
  static constexpr size_t BYTES = 1024 + CTRL_OFF + 256;
  static_assert(BYTES <= 227 * 1024, "attn_loop_kernel: shared memory");
};

template <int HDP>
__global__ void __launch_bounds__(AL_THREADS, 1)
    attn_loop_kernel(const __grid_constant__ CUtensorMap tmap_qkv, const __grid_constant__ CUtensorMap tmap_qkv_b,
                     const __grid_constant__ CUtensorMap tmap_bias, const __grid_constant__ AttnLoopParams p) {
  using SM = AttnLoopSmem<HDP>;
  using HT = HeadTile<HDP>;
  constexpr int TILE_BYTES = SM::TILE_BYTES;
  constexpr int NKV = SM::NKV, NB = AL_NB, BUNIT = AL_BUNIT;
  constexpr int BUNIT_BYTES = SM::BUNIT_BYTES;
  constexpr int UNITS = 128 / BUNIT;              // bias units per key tile
  constexpr int O_LD = SM::O_LD;
  constexpr int Q_OFF = SM::Q_OFF, KV_OFF = SM::KV_OFF, P_OFF = SM::P_OFF, BIAS_OFF = SM::BIAS_OFF;
  constexpr int SACC_OFF = SM::SACC_OFF, OACC_OFF = SM::OACC_OFF, CTRL_OFF = SM::CTRL_OFF;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int S = p.S, nkt = p.nkt;
  float* sacc = reinterpret_cast<float*>(smem + SACC_OFF);
  float* oacc = reinterpret_cast<float*>(smem + OACC_OFF);
  uint64_t* q_full = reinterpret_cast<uint64_t*>(smem + CTRL_OFF);
  uint64_t* q_empty = q_full + 1;
  uint64_t* kv_full = q_empty + 1;         // [NKV]
  uint64_t* kv_empty = kv_full + NKV;      // [NKV]
  uint64_t* b_full = kv_empty + NKV;       // [NB]
  uint64_t* b_empty = b_full + NB;         // [NB]

  if (warp == AL_PRODUCER && lane == 0) {
    tma_prefetch_desc(&tmap_qkv);
    if (HT::HB > 0) tma_prefetch_desc(&tmap_qkv_b);
    if (p.has_bias) tma_prefetch_desc(&tmap_bias);
    mbar_init(q_full, 1), mbar_init(q_empty, 1);
    for (int i = 0; i < NKV; ++i) mbar_init(&kv_full[i], 1), mbar_init(&kv_empty[i], 1);
    for (int i = 0; i < NB; ++i) mbar_init(&b_full[i], 1), mbar_init(&b_empty[i], 4);
    fence_mbar_init();
  }
  __syncthreads();

  const int items = p.groups * p.heads * p.nqt;
  // item -> (head, q tile) outer, window inner: CTAs running side by side share the bias tiles in L2
  auto decode = [&](int w, int& grp, int& head, int& qi) {
    grp = w % p.groups;
    const int hq = w / p.groups;
    qi = hq % p.nqt;
    head = hq / p.nqt;
  };
  auto units_of = [&](int j) { return min(UNITS, (min(128, S - j * 128) + BUNIT - 1) / BUNIT); };  // live bias units of key tile j

  if (warp == AL_PRODUCER) {
    if (lane == 0) {
      uint32_t kv_cnt = 0, b_cnt = 0, it = 0;
      auto load_kv = [&](int which, int j, int row0, int head) {
        const int st = kv_cnt % NKV;
        mbar_wait(&kv_empty[st], ((kv_cnt / NKV) & 1) ^ 1);
        mbar_expect_tx(&kv_full[st], TILE_BYTES);
        HT::load(smem + KV_OFF + st * TILE_BYTES, AL_ROWS, 0, &tmap_qkv, &tmap_qkv_b, &kv_full[st],
                 (which * p.heads + head) * HDP, row0 + j * 128);
        ++kv_cnt;
      };
      for (int w = blockIdx.x; w < items; w += gridDim.x, ++it) {
        int grp, head, qi;
        decode(w, grp, head, qi);
        const int row0 = grp * S;
        mbar_wait(q_empty, (it & 1) ^ 1);
        mbar_expect_tx(q_full, TILE_BYTES);
        HT::load(smem + Q_OFF, AL_ROWS, 0, &tmap_qkv, &tmap_qkv_b, q_full, head * HDP, row0 + qi * 128);
        // consumption order: pass 1 K_0 b_0 K_1 b_1 ...; pass 2 K_0 b_0 V_0 K_1 b_1 V_1 ...
        for (int pass = 0; pass < 2; ++pass) {
          for (int j = 0; j < nkt; ++j) {
            load_kv(1, j, row0, head);
            if (p.has_bias) {
              for (int u = 0; u < units_of(j); ++u) {
                const int bs = b_cnt % NB;
                mbar_wait(&b_empty[bs], ((b_cnt / NB) & 1) ^ 1);
                mbar_expect_tx(&b_full[bs], BUNIT_BYTES);
                tma_load_2d(smem + BIAS_OFF + bs * BUNIT_BYTES, &tmap_bias, &b_full[bs], j * 128 + u * BUNIT,
                            head * S + qi * 128);
                ++b_cnt;
              }
            }
            if (pass == 1) load_kv(2, j, row0, head);
          }
        }
      }
    }
  } else {
    const int quad = warp & 3;
    const int r = quad * 32 + lane;  // query row inside the tile
    const int tid = threadIdx.x;
    uint8_t* sP = smem + P_OFF;
    const uint32_t sQ = smem_u32(smem + Q_OFF);
    const uint32_t sPu = smem_u32(sP);
    const float* arow = sacc + r * AL_ACC_LD;
    uint32_t kv_cnt = 0, b_cnt = 0, it = 0;
    const bool use_bias = p.has_bias != 0;
    // S_j = Q K_j^T from the next ring stage into the score tile (the stage is released once the MMAs are done)
    auto score_mma = [&](bool last_of_item) {
      const int st = kv_cnt % NKV;
      mbar_wait(&kv_full[st], (kv_cnt / NKV) & 1);
      const uint32_t sK = smem_u32(smem + KV_OFF + st * TILE_BYTES);
      named_bar_sync(1, 128);  // every read of the previous score tile is done
      wg_mma_128<128, 0, 0, HT::KSTEPS>(
          sacc, AL_ACC_LD, [&](int h, int k) { return HT::kdesc(sQ, AL_ROWS, h * 64, k); },
          [&](int k) { return HT::kdesc(sK, AL_ROWS, 0, k); }, false);
      named_bar_sync(1, 128);
      if (tid == 0) {
        mbar_arrive(&kv_empty[st]);
        if (last_of_item) mbar_arrive(q_empty);
      }
      ++kv_cnt;
    };
    for (int w = blockIdx.x; w < items; w += gridDim.x, ++it) {
      int grp, head, qi;
      decode(w, grp, head, qi);
      const int qrow = qi * 128 + r;
      const bool row_ok = qrow < S;
      float mx = -INFINITY, sum = 0.f;
      mbar_wait(q_full, it & 1);
      for (int pass = 0; pass < 2; ++pass) {
        for (int j = 0; j < nkt; ++j) {
          score_mma(pass == 1 && j == nkt - 1);
          const int ncols = min(128, S - j * 128);  // valid keys of this tile
          for (int u = 0; u < UNITS; ++u) {
            const bool unit_live = u * BUNIT < ncols;
            const uint8_t* bunit = nullptr;
            if (use_bias && unit_live) {
              const int bs = b_cnt % NB;
              mbar_wait(&b_full[bs], (b_cnt / NB) & 1);
              bunit = smem + BIAS_OFF + bs * BUNIT_BYTES;
            }
            const int c0 = u * BUNIT;  // first key column of this 32-wide chunk
            if (pass == 1 || c0 < ncols) {
              uint32_t raw[32];
              float sc[32];
              if (c0 < ncols) {
                ld_row32(arow + c0, raw);
                const uint8_t* brow = bunit ? bunit + r * 128 : nullptr;
#pragma unroll
                for (int q4 = 0; q4 < 8; ++q4) {
                  float4 b4 = make_float4(0.f, 0.f, 0.f, 0.f);
                  if (brow) b4 = *reinterpret_cast<const float4*>(brow + ((q4 ^ (r & 7)) << 4));
                  const float bb[4] = {b4.x, b4.y, b4.z, b4.w};
#pragma unroll
                  for (int e = 0; e < 4; ++e) {
                    const int c = q4 * 4 + e;
                    const float v = fmaf(__uint_as_float(raw[c]), p.scale_log2e, bb[e] * 1.4426950408889634f);
                    sc[c] = (c0 + c < ncols) ? v : -INFINITY;
                  }
                }
              } else {
#pragma unroll
                for (int c = 0; c < 32; ++c) sc[c] = -INFINITY;
              }
              if (pass == 0) {
#pragma unroll
                for (int c = 0; c < 32; ++c) mx = fmaxf(mx, sc[c]);
              } else {
                uint32_t pk[16];
#pragma unroll
                for (int c = 0; c < 32; c += 2) {
                  const float e0 = row_ok ? exp2f(sc[c] - mx) : 0.f;  // exp2(-inf) = 0 for masked keys
                  const float e1 = row_ok ? exp2f(sc[c + 1] - mx) : 0.f;
                  const __half2 hh = __floats2half2_rn(e0, e1);
                  sum += __low2float(hh) + __high2float(hh);  // what the tensor core will multiply
                  pk[c >> 1] = *reinterpret_cast<const uint32_t*>(&hh);
                }
#pragma unroll
                for (int q = 0; q < 4; ++q) {
                  const int c = c0 + q * 8;
                  *reinterpret_cast<uint4*>(sP + (c >> 6) * (AL_ROWS * 128) + r * 128 + ((((c & 63) >> 3) ^ (r & 7)) << 4)) =
                      make_uint4(pk[4 * q], pk[4 * q + 1], pk[4 * q + 2], pk[4 * q + 3]);
                }
              }
            }
            if (use_bias && unit_live) {
              __syncwarp();
              if (lane == 0) mbar_arrive(&b_empty[b_cnt % NB]);
              ++b_cnt;
            }
          }
          if (pass == 0 && !row_ok) mx = 0.f;
          if (pass == 1) {
            // O (+)= P_j V_j: P is complete once every thread has written its row
            fence_proxy_async_smem();
            named_bar_sync(1, 128);
            const int st = kv_cnt % NKV;
            mbar_wait(&kv_full[st], (kv_cnt / NKV) & 1);
            const uint32_t sV = smem_u32(smem + KV_OFF + st * TILE_BYTES);
            wg_mma_128_head<HDP, 0, 8>(
                oacc, O_LD,
                [&](int h, int ks) {
                  return make_smem_desc(sPu + (ks >> 2) * (AL_ROWS * 128) + h * 64 * 128 + (ks & 3) * 32, 16, 1024, SWZ_128B);
                },
                sV, AL_ROWS, j > 0);
            named_bar_sync(1, 128);  // P V complete: V stage and P tile are free, O rows are readable
            if (tid == 0) mbar_arrive(&kv_empty[st]);
            ++kv_cnt;
          }
        }
        if (pass == 0 && !row_ok) mx = 0.f;
      }
      // O epilogue
      const float inv = row_ok ? 1.f / sum : 0.f;
      const long long grow = (long long)grp * S + qrow;
      if (row_ok) store_row_f16<HDP>(oacc + r * O_LD, inv, p.out + grow * p.ldo + head * HDP);
      if (p.lse && row_ok) p.lse[grow * p.heads + head] = mx + log2f(sum);
    }
  }
}

template <int HDP>
static int launch_attn_loop(const CUtensorMap& tq, const CUtensorMap& tqb, const CUtensorMap& tb, const AttnLoopParams& p,
                            cudaStream_t st) {
  constexpr size_t smem = AttnLoopSmem<HDP>::BYTES;
  static bool configured = false;
  if (!configured) {
    FVIT_CUDA(cudaFuncSetAttribute(attn_loop_kernel<HDP>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    configured = true;
  }
  const long long items = (long long)p.groups * p.heads * p.nqt;
  const int slots = num_sms();
  attn_loop_kernel<HDP><<<(unsigned)(items < slots ? items : slots), AL_THREADS, smem, st>>>(tq, tqb, tb, p);
  return post_launch("attn_loop_kernel");
}

}  // namespace fvit

using namespace fvit;

extern "C" int fvit_attn_loop_fwd(const void* qkv, int64_t ldq, int32_t groups, int32_t S, int32_t heads, int32_t hdp,
                                  const float* bias, float scale, void* out, int64_t ldo, float* lse, void* stream) {
  FVIT_CHECK(qkv && out && groups > 0 && heads > 0, "fvit_attn_loop_fwd: bad arguments");
  // (any S: one tile is the case nqt = nkt = 1. Inference plans give windows of up to 128 tokens to fvit_attn_tc_fwd / the fused
  // kernel, which pack several windows into a tile; training plans come here from 65 tokens on for the log-sum-exp rows)
  FVIT_CHECK(S > 0, "fvit_attn_loop_fwd: S=%d", S);
  FVIT_CHECK(hdp == 32 || hdp == 64 || hdp == 80, "fvit_attn_loop_fwd: padded head dim %d unsupported (32, 64 or 80)",
             hdp);
  FVIT_CHECK(ldq % 8 == 0 && ldo % 8 == 0 && ldq >= 3 * heads * hdp && ldo >= heads * hdp,
             "fvit_attn_loop_fwd: bad leading dimensions");
  FVIT_CHECK(!bias || S % 4 == 0, "fvit_attn_loop_fwd: the bias rows of S=%d tokens are not 16-byte aligned (TMA)", S);
  FVIT_CHECK((reinterpret_cast<uintptr_t>(out) & 15) == 0, "fvit_attn_loop_fwd: out must be 16-byte aligned");
  AttnLoopParams p;
  p.groups = groups, p.S = S, p.heads = heads;
  p.nqt = p.nkt = (S + 127) / 128;
  p.scale_log2e = scale * 1.4426950408889634f;
  p.has_bias = bias ? 1 : 0;
  p.out = (__half*)out, p.ldo = ldo, p.lse = lse;
  CUtensorMap tq, tqb, tb;
  {
    int rc = head_tile_tmaps(&tq, &tqb, qkv, 3 * heads * hdp, (uint64_t)groups * S, ldq, hdp, AL_ROWS);
    if (rc) return rc;
  }
  if (bias) {
    uint64_t dims[2] = {(uint64_t)S, (uint64_t)heads * S};
    uint64_t strides[1] = {(uint64_t)S * 4};
    uint32_t box[2] = {32, (uint32_t)AL_ROWS};
    int rc = cached_tmap_f32(&tb, bias, 2, dims, strides, box, CU_TENSOR_MAP_SWIZZLE_128B);
    if (rc) return rc;
  } else {
    tb = tq;
  }
  if (hdp == 80) return launch_attn_loop<80>(tq, tqb, tb, p, (cudaStream_t)stream);
  if (hdp == 64) return launch_attn_loop<64>(tq, tqb, tb, p, (cudaStream_t)stream);
  return launch_attn_loop<32>(tq, tqb, tb, p, (cudaStream_t)stream);
}

// =====================================================================================================
// fvit_attn_loop_bwd_long: tensor-core backward of the attention core for windows longer than one tile (S > 128: any-res
// S = 148, the 21k models' 14 x 14 ... 48 x 48 windows, fv.py:1253-1418). Work item = (window, head); with lse (forward)
// and delta = rowsum(dO * O) per query row, key tiles j outside, query tiles i inside:
//   S = Q_i K_j^T, dP = dO_i V_j^T     (wgmma, in two 64-key halves through fp32 shared-memory tiles)
//   P = exp2(S*scale*log2e + bias*log2e - lse), dS = P*(dP - delta)   (one thread per query row; fp16 tiles in shared
//       memory; dS accumulated into dbias with 16-byte reductions)
//   dV_j += P^T dO_i, dK_j += dS^T Q_i (register accumulators of the warpgroup over the query loop)
//   and the PARTIAL dQ_i = dS K_j of this pair (not accumulated: nt tiles of dQ do not fit on chip).
// The thread that owns query row r of every tile adds the partial to its row of an fp32 scratch matrix
// dq_scratch[groups * S, heads * HDP] (plain 16-byte stores for j = 0, 16-byte reductions afterwards) and converts
// the row to fp16 once the key loop is over. Only one CTA ever touches a (window, head) slice and only one thread a
// row of it, so the reductions need no initialisation and no ordering beyond program order. Q_i / dO_i stream through
// the operand ring (L2 hits after the first key tile); delta and the log-sum-exp rows sit in shared memory.
//   warp 4     : TMA producer (K_j / V_j, then Q_i / dO_i for every i, in consumption order)
//   warps 0..3 : one warpgroup: every MMA, the softmax gradient and the epilogues
namespace fvit {

struct AttnLoopBwdParams {
  int groups, S, heads, nt;
  float scale, scale_log2e;
  const float* bias;
  float* dbias;
  const float* lse;
  const __half* dout;
  long long lddo;
  const __half* out;
  long long ldo;
  __half* dqkv;
  long long lddq;
};

struct AttnLoopBwdLongParams {
  AttnLoopBwdParams b;
  float* dq32;
  long long lddq32;
};

constexpr int ALL_THREADS = AL_THREADS;
constexpr int ALL_HALF_LD = 68;  // floats per row of the 64-column fp32 score / dP tiles

template <int HDP>
struct AttnBwdLongSmem {
  static constexpr int TILE_BYTES = AL_ROWS * HDP * 2;
  static constexpr int NQ = HDP == 32 ? 2 : 1;              // (Q_i, dO_i) ring depth
  static constexpr int QDO_OFF = 0;
  static constexpr int KV_OFF = NQ * 2 * TILE_BYTES;        // one (K_j, V_j) stage
  static constexpr int P_OFF = KV_OFF + 2 * TILE_BYTES;
  static constexpr int DS_OFF = P_OFF + AL_ROWS * 128 * 2;
  static constexpr int WORK_OFF = DS_OFF + AL_ROWS * 128 * 2;  // S / dP halves, dQ partial, dK / dV staging
  static constexpr int WORK_BYTES = 2 * AL_ROWS * ALL_HALF_LD * 4;
  static constexpr int CTRL_OFF = WORK_OFF + WORK_BYTES;
  static constexpr int ROWV_OFF = CTRL_OFF + 256;           // delta[nt * 128], lse[nt * 128]
  static_assert(AL_ROWS * (HDP + 4) * 4 <= WORK_BYTES, "dQ / dK / dV staging fits the work area");
};

template <int HDP>
__global__ void __launch_bounds__(ALL_THREADS, 1)
    attn_loop_bwd_long_kernel(const __grid_constant__ CUtensorMap tmap_qkv, const __grid_constant__ CUtensorMap tmap_do,
                              const __grid_constant__ CUtensorMap tmap_qkv_b, const __grid_constant__ CUtensorMap tmap_do_b,
                              const __grid_constant__ AttnLoopBwdLongParams pl) {
  using SM = AttnBwdLongSmem<HDP>;
  using HT = HeadTile<HDP>;
  constexpr int HA = HT::HA, HB = HT::HB;
  const AttnLoopBwdParams& p = pl.b;
  constexpr int TILE_BYTES = SM::TILE_BYTES;
  constexpr int NQ = SM::NQ;
  constexpr int G_LD = HDP + 4;  // row stride of the dQ / dK / dV fp32 tiles
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int S = p.S, nt = p.nt;
  uint64_t* qdo_full = reinterpret_cast<uint64_t*>(smem + SM::CTRL_OFF);  // [2]
  uint64_t* qdo_empty = qdo_full + 2;  // [2]
  uint64_t* kv_full = qdo_empty + 2;
  uint64_t* kv_empty = kv_full + 1;
  float* s_delta = reinterpret_cast<float*>(smem + SM::ROWV_OFF);
  float* s_lse = s_delta + nt * 128;
  float* work = reinterpret_cast<float*>(smem + SM::WORK_OFF);
  float* s_half = work;                                // S[:, 64c .. 64c + 64)
  float* dp_half = work + AL_ROWS * ALL_HALF_LD;       // dP[:, 64c .. 64c + 64)

  if (warp == AL_PRODUCER && lane == 0) {
    tma_prefetch_desc(&tmap_qkv);
    tma_prefetch_desc(&tmap_do);
    if (HB > 0) tma_prefetch_desc(&tmap_qkv_b), tma_prefetch_desc(&tmap_do_b);
    for (int i = 0; i < 2; ++i) mbar_init(&qdo_full[i], 1), mbar_init(&qdo_empty[i], 1);
    mbar_init(kv_full, 1), mbar_init(kv_empty, 1);
    fence_mbar_init();
  }
  __syncthreads();

  const int items = p.groups * p.heads;

  if (warp == AL_PRODUCER) {
    if (lane == 0) {
      uint32_t kv_cnt = 0, pair = 0;
      for (int w = blockIdx.x; w < items; w += gridDim.x) {
        const int grp = w % p.groups, head = w / p.groups;
        const int row0 = grp * S;
        for (int j = 0; j < nt; ++j, ++kv_cnt) {
          mbar_wait(kv_empty, (kv_cnt & 1) ^ 1);
          mbar_expect_tx(kv_full, 2 * TILE_BYTES);
          HT::load(smem + SM::KV_OFF, AL_ROWS, 0, &tmap_qkv, &tmap_qkv_b, kv_full, (p.heads + head) * HDP, row0 + j * 128);
          HT::load(smem + SM::KV_OFF + TILE_BYTES, AL_ROWS, 0, &tmap_qkv, &tmap_qkv_b, kv_full, (2 * p.heads + head) * HDP,
                   row0 + j * 128);
          for (int i = 0; i < nt; ++i, ++pair) {
            const int qs = pair % NQ;
            mbar_wait(&qdo_empty[qs], ((pair / NQ) & 1) ^ 1);
            mbar_expect_tx(&qdo_full[qs], 2 * TILE_BYTES);
            HT::load(smem + SM::QDO_OFF + (2 * qs) * TILE_BYTES, AL_ROWS, 0, &tmap_qkv, &tmap_qkv_b, &qdo_full[qs],
                     head * HDP, row0 + i * 128);
            HT::load(smem + SM::QDO_OFF + (2 * qs + 1) * TILE_BYTES, AL_ROWS, 0, &tmap_do, &tmap_do_b, &qdo_full[qs],
                     head * HDP, row0 + i * 128);
          }
        }
      }
    }
  } else {
    const int quad = warp & 3;
    const int r = quad * 32 + lane;
    const int tid = threadIdx.x;
    uint8_t* sP = smem + SM::P_OFF;
    uint8_t* sDS = smem + SM::DS_OFF;
    const uint32_t sPu = smem_u32(sP), sDSu = smem_u32(sDS);
    const uint32_t sK = smem_u32(smem + SM::KV_OFF), sV = sK + TILE_BYTES;
    uint32_t kv_cnt = 0, pair = 0;
    const int Cp = p.heads * HDP;
    for (int w = blockIdx.x; w < items; w += gridDim.x) {
      const int grp = w % p.groups, head = w / p.groups;
      const long long row0 = (long long)grp * S;
      // per query row: delta = sum_c dO * O and the forward's log-sum-exp
      named_bar_sync(1, 128);  // the previous item's readers of the row vectors are done
      for (int i = 0; i < nt; ++i) {
        const int q = i * 128 + r;
        float acc = 0.f, l = 0.f;
        if (q < S) {
          const uint4* a = reinterpret_cast<const uint4*>(p.dout + (row0 + q) * p.lddo + head * HDP);
          const uint4* b = reinterpret_cast<const uint4*>(p.out + (row0 + q) * p.ldo + head * HDP);
#pragma unroll
          for (int v = 0; v < HDP / 8; ++v) {
            const uint4 x = __ldg(a + v), y = __ldg(b + v);
            const __half2* hx = reinterpret_cast<const __half2*>(&x);
            const __half2* hy = reinterpret_cast<const __half2*>(&y);
#pragma unroll
            for (int e = 0; e < 4; ++e) {
              const float2 fx = __half22float2(hx[e]), fy = __half22float2(hy[e]);
              acc = fmaf(fx.x, fy.x, fmaf(fx.y, fy.y, acc));
            }
          }
          l = p.lse[(row0 + q) * p.heads + head];
        }
        s_delta[q] = acc, s_lse[q] = l;
      }
      for (int j = 0; j < nt; ++j, ++kv_cnt) {
        const int ncols = min(128, S - j * 128);
        mbar_wait(kv_full, kv_cnt & 1);
        // dV_j / dK_j accumulators (rows 64h .. 64h + 63 = keys of this tile), summed over the query tiles: head
        // columns [0, HA) in dv / dk, [HA, HDP) in dvb / dkb
        float dv[2][HA / 2], dk[2][HA / 2], dvb[2][HB > 0 ? HB / 2 : 1], dkb[2][HB > 0 ? HB / 2 : 1];
#pragma unroll
        for (int h = 0; h < 2; ++h) {
#pragma unroll
          for (int u = 0; u < HA / 2; ++u) dv[h][u] = 0.f, dk[h][u] = 0.f;
#pragma unroll
          for (int u = 0; u < (HB > 0 ? HB / 2 : 1); ++u) dvb[h][u] = 0.f, dkb[h][u] = 0.f;
        }
        for (int i = 0; i < nt; ++i, ++pair) {
          const int qs = pair % NQ;
          mbar_wait(&qdo_full[qs], (pair / NQ) & 1);
          const uint32_t sQ = smem_u32(smem + SM::QDO_OFF + (2 * qs) * TILE_BYTES), sDO = sQ + TILE_BYTES;
          const int q = i * 128 + r;
          const bool row_ok = q < S;
          const float my_lse = s_lse[q], my_delta = s_delta[q];
          const float* brow = (p.bias && row_ok) ? p.bias + ((long long)head * S + q) * S + j * 128 : nullptr;
          float* dbrow = (p.dbias && row_ok) ? p.dbias + ((long long)head * S + q) * S + j * 128 : nullptr;
#pragma unroll 1
          for (int ch = 0; ch < 2; ++ch) {  // key columns [64ch, 64ch + 64) of the pair
            named_bar_sync(1, 128);         // the work area is free
            wg_mma_128<64, 0, 0, HT::KSTEPS>(
                s_half, ALL_HALF_LD, [&](int h, int k) { return HT::kdesc(sQ, AL_ROWS, h * 64, k); },
                [&](int k) { return HT::kdesc(sK, AL_ROWS, ch * 64, k); }, false);
            wg_mma_128<64, 0, 0, HT::KSTEPS>(
                dp_half, ALL_HALF_LD, [&](int h, int k) { return HT::kdesc(sDO, AL_ROWS, h * 64, k); },
                [&](int k) { return HT::kdesc(sV, AL_ROWS, ch * 64, k); }, false);
            named_bar_sync(1, 128);
#pragma unroll 1
            for (int cc = 0; cc < 64; cc += 16) {
              const int c0 = ch * 64 + cc;
              uint32_t pkp[8], pkd[8];
              if (c0 < ncols) {
                uint32_t rs[16], rd[16];
                ld_row16(s_half + r * ALL_HALF_LD + cc, rs);
                ld_row16(dp_half + r * ALL_HALF_LD + cc, rd);
#pragma unroll
                for (int q4 = 0; q4 < 4; ++q4) {
                  const int c = c0 + q4 * 4;
                  const float4 b4 =
                      (brow && c < ncols) ? __ldg(reinterpret_cast<const float4*>(brow + c)) : make_float4(0.f, 0.f, 0.f, 0.f);
                  const float bb[4] = {b4.x, b4.y, b4.z, b4.w};
                  float pv[4], ds[4];
#pragma unroll
                  for (int e = 0; e < 4; ++e) {
                    const bool in = row_ok && (c + e < ncols);
                    const float sc = fmaf(__uint_as_float(rs[q4 * 4 + e]), p.scale_log2e, fmaf(bb[e], 1.4426950408889634f, -my_lse));
                    pv[e] = in ? exp2f(sc) : 0.f;
                    ds[e] = in ? pv[e] * (__uint_as_float(rd[q4 * 4 + e]) - my_delta) : 0.f;
                  }
                  if (dbrow && c < ncols)  // (S % 4 == 0: a 4-column group is entirely inside or outside the window)
                    asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(dbrow + c), "f"(ds[0]), "f"(ds[1]),
                                 "f"(ds[2]), "f"(ds[3])
                                 : "memory");
                  const __half2 p0 = __floats2half2_rn(pv[0], pv[1]), p1 = __floats2half2_rn(pv[2], pv[3]);
                  const __half2 d0 = __floats2half2_rn(ds[0], ds[1]), d1 = __floats2half2_rn(ds[2], ds[3]);
                  pkp[q4 * 2] = *reinterpret_cast<const uint32_t*>(&p0), pkp[q4 * 2 + 1] = *reinterpret_cast<const uint32_t*>(&p1);
                  pkd[q4 * 2] = *reinterpret_cast<const uint32_t*>(&d0), pkd[q4 * 2 + 1] = *reinterpret_cast<const uint32_t*>(&d1);
                }
              } else {
#pragma unroll
                for (int e = 0; e < 8; ++e) pkp[e] = 0u, pkd[e] = 0u;
              }
#pragma unroll
              for (int qq = 0; qq < 2; ++qq) {
                const int c = c0 + qq * 8;
                const uint32_t off = (c >> 6) * (AL_ROWS * 128) + r * 128 + ((((c & 63) >> 3) ^ (r & 7)) << 4);
                *reinterpret_cast<uint4*>(sP + off) = make_uint4(pkp[4 * qq], pkp[4 * qq + 1], pkp[4 * qq + 2], pkp[4 * qq + 3]);
                *reinterpret_cast<uint4*>(sDS + off) = make_uint4(pkd[4 * qq], pkd[4 * qq + 1], pkd[4 * qq + 2], pkd[4 * qq + 3]);
              }
            }
          }
          fence_proxy_async_smem();
          named_bar_sync(1, 128);  // P / dS complete, S / dP reads done
          // dV_j += P^T dO_i, dK_j += dS^T Q_i: A read MN-major (M = keys, K = 128 query rows)
          wgmma_fence();
#pragma unroll
          for (int h = 0; h < 2; ++h) {
#pragma unroll
            for (int ks = 0; ks < 8; ++ks) {
              const uint64_t ap = make_smem_desc(sPu + h * (AL_ROWS * 128) + ks * 2048, AL_ROWS * 128, 1024, SWZ_128B);
              const uint64_t ads = make_smem_desc(sDSu + h * (AL_ROWS * 128) + ks * 2048, AL_ROWS * 128, 1024, SWZ_128B);
              Wgmma<HA, 1, 1, 0>::mma(dv[h], ap, HT::ndesc_a(sDO, ks), 1u);
              Wgmma<HA, 1, 1, 0>::mma(dk[h], ads, HT::ndesc_a(sQ, ks), 1u);
              if constexpr (HB > 0) {
                Wgmma<HB, 1, 1, 0>::mma(dvb[h], ap, HT::ndesc_b(sDO, AL_ROWS, ks), 1u);
                Wgmma<HB, 1, 1, 0>::mma(dkb[h], ads, HT::ndesc_b(sQ, AL_ROWS, ks), 1u);
              }
            }
          }
          wgmma_commit();
          wgmma_wait0();
          // partial dQ_i = dS K_j into the work area, then this thread's row into the fp32 scratch
          wg_mma_128_head<HDP, 0, 8>(
              work, G_LD,
              [&](int h, int ks) {
                return make_smem_desc(sDSu + (ks >> 2) * (AL_ROWS * 128) + h * 64 * 128 + (ks & 3) * 32, 16, 1024, SWZ_128B);
              },
              sK, AL_ROWS, false);
          named_bar_sync(1, 128);
          if (tid == 0) mbar_arrive(&qdo_empty[qs]);  // Q_i / dO_i consumed
          if (row_ok) {
            float* drow = pl.dq32 + (row0 + q) * pl.lddq32 + head * HDP;
            const float* arow = work + r * G_LD;
#pragma unroll
            for (int c0 = 0; c0 < HDP; c0 += 4) {
              const float4 a = *reinterpret_cast<const float4*>(arow + c0);
              const float v0 = a.x * p.scale, v1 = a.y * p.scale, v2 = a.z * p.scale, v3 = a.w * p.scale;
              if (j == 0)
                *reinterpret_cast<float4*>(drow + c0) = make_float4(v0, v1, v2, v3);
              else
                asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(drow + c0), "f"(v0), "f"(v1), "f"(v2),
                             "f"(v3)
                             : "memory");
            }
          }
        }
        // every MMA of this key tile is complete: K_j / V_j are free; dK_j, then dV_j (row r = key j*128 + r) through the
        // work area
        named_bar_sync(1, 128);
        if (tid == 0) mbar_arrive(kv_empty);
        {
          const int key = j * 128 + r;
          __half* orow = p.dqkv + (row0 + key) * p.lddq + head * HDP;
#pragma unroll
          for (int which = 1; which < 3; ++which) {
            if (which == 2) named_bar_sync(1, 128);  // every dK row is read: dV overwrites the work area
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              acc_store<HA>(work + h * 64 * G_LD, G_LD, which == 1 ? dk[h] : dv[h]);
              if constexpr (HB > 0) acc_store<HB>(work + h * 64 * G_LD + HA, G_LD, which == 1 ? dkb[h] : dvb[h]);
            }
            named_bar_sync(1, 128);
            if (key < S) store_row_f16<HDP>(work + r * G_LD, which == 1 ? p.scale : 1.f, orow + which * Cp);
          }
        }
      }
      // dQ rows of this (window, head): fp32 scratch (each row written by this thread only) -> fp16
      __threadfence();
      for (int i = 0; i < nt; ++i) {
        const int q = i * 128 + r;
        if (q < S) {
          const float* drow = pl.dq32 + (row0 + q) * pl.lddq32 + head * HDP;
          __half* orow = p.dqkv + (row0 + q) * p.lddq + head * HDP;
#pragma unroll
          for (int c = 0; c < HDP; c += 8) {
            const float4 a = __ldcg(reinterpret_cast<const float4*>(drow + c));
            const float4 b = __ldcg(reinterpret_cast<const float4*>(drow + c + 4));
            const __half2 h0 = __floats2half2_rn(a.x, a.y), h1 = __floats2half2_rn(a.z, a.w);
            const __half2 h2 = __floats2half2_rn(b.x, b.y), h3 = __floats2half2_rn(b.z, b.w);
            *reinterpret_cast<uint4*>(orow + c) =
                make_uint4(*reinterpret_cast<const uint32_t*>(&h0), *reinterpret_cast<const uint32_t*>(&h1),
                           *reinterpret_cast<const uint32_t*>(&h2), *reinterpret_cast<const uint32_t*>(&h3));
          }
        }
      }
    }
  }
}

template <int HDP>
static int launch_attn_loop_bwd_long(const CUtensorMap& tq, const CUtensorMap& td, const CUtensorMap& tqb,
                                     const CUtensorMap& tdb, const AttnLoopBwdLongParams& p, cudaStream_t st) {
  const size_t smem = 1024 + (size_t)AttnBwdLongSmem<HDP>::ROWV_OFF + (size_t)p.b.nt * 128 * 8;
  FVIT_CHECK(smem <= 227 * 1024, "fvit_attn_loop_bwd_long: S=%d needs %zu bytes of shared memory", p.b.S, smem);
  static size_t configured = 0;
  if (smem > configured) {
    FVIT_CUDA(cudaFuncSetAttribute(attn_loop_bwd_long_kernel<HDP>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    configured = smem;
  }
  const int items = p.b.groups * p.b.heads;
  const int sms = num_sms();
  attn_loop_bwd_long_kernel<HDP><<<items < sms ? items : sms, ALL_THREADS, smem, st>>>(tq, td, tqb, tdb, p);
  return post_launch("attn_loop_bwd_long_kernel");
}

}  // namespace fvit

extern "C" int fvit_attn_loop_bwd_long(const void* qkv, int64_t ldq, const void* dout, int64_t lddo, const void* out,
                                       int64_t ldo, const float* lse, int32_t groups, int32_t S, int32_t heads, int32_t hdp,
                                       const float* bias, float scale, void* dqkv, int64_t lddq, float* dbias,
                                       float* dq_scratch, int64_t ld_scratch, void* stream) {
  using namespace fvit;
  FVIT_CHECK(qkv && dout && out && lse && dqkv && dq_scratch && groups > 0 && heads > 0, "fvit_attn_loop_bwd_long: bad arguments");
  FVIT_CHECK(S > 0, "fvit_attn_loop_bwd_long: S=%d", S);
  FVIT_CHECK(S % 4 == 0, "fvit_attn_loop_bwd_long: S=%d must be a multiple of 4 (16-byte bias / dbias accesses)", S);
  FVIT_CHECK(hdp == 32 || hdp == 64 || hdp == 80, "fvit_attn_loop_bwd_long: padded head dim %d unsupported", hdp);
  FVIT_CHECK(ldq % 8 == 0 && lddo % 8 == 0 && ldo % 8 == 0 && lddq % 8 == 0 && ld_scratch % 4 == 0 &&
                 ld_scratch >= (int64_t)heads * hdp && (reinterpret_cast<uintptr_t>(dq_scratch) & 15) == 0,
             "fvit_attn_loop_bwd_long: bad leading dimensions");
  AttnLoopBwdLongParams pl;
  AttnLoopBwdParams& p = pl.b;
  p.groups = groups, p.S = S, p.heads = heads, p.nt = (S + 127) / 128;
  p.scale = scale, p.scale_log2e = scale * 1.4426950408889634f;
  p.bias = bias, p.dbias = dbias, p.lse = lse;
  p.dout = (const __half*)dout, p.lddo = lddo, p.out = (const __half*)out, p.ldo = ldo;
  p.dqkv = (__half*)dqkv, p.lddq = lddq;
  pl.dq32 = dq_scratch, pl.lddq32 = ld_scratch;
  CUtensorMap tq, td, tqb, tdb;
  int rc = head_tile_tmaps(&tq, &tqb, qkv, 3 * heads * hdp, (uint64_t)groups * S, ldq, hdp, AL_ROWS);
  if (rc) return rc;
  rc = head_tile_tmaps(&td, &tdb, dout, heads * hdp, (uint64_t)groups * S, lddo, hdp, AL_ROWS);
  if (rc) return rc;
  if (hdp == 80) return launch_attn_loop_bwd_long<80>(tq, td, tqb, tdb, pl, (cudaStream_t)stream);
  if (hdp == 64) return launch_attn_loop_bwd_long<64>(tq, td, tqb, tdb, pl, (cudaStream_t)stream);
  return launch_attn_loop_bwd_long<32>(tq, td, tqb, tdb, pl, (cudaStream_t)stream);
}
