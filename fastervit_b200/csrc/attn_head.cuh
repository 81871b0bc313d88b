// Shared-memory layout of one head's Q / K / V / dO rows in the tensor-core attention kernels, for padded head dims
// HDP = 32, 64 and 80.
//
// A head tile holds R rows of HDP fp16 columns as swizzled atoms that TMA writes and wgmma reads directly:
//   HDP 32 : one atom of 64-byte rows, 64B swizzle
//   HDP 64 : one atom of 128-byte rows, 128B swizzle
//   HDP 80 : columns [0, 64) as a 128B-swizzled atom of 128-byte rows, then columns [64, 80) as a 32B-swizzled atom of
//            32-byte rows (a 160-byte row is no swizzle atom). Two TMA boxes per tile, from two tensor maps over the
//            same matrix; a K = head-dim product is four k16 steps on the first atom and one on the second, an
//            N = head-dim product an n64 and an n16 wgmma.
#pragma once
#include <cuda_fp16.h>

#include "common.h"
#include "ptx.cuh"
#include "wgmma.cuh"

namespace fvit {

template <int HDP>
struct HeadTile {
  static_assert(HDP == 32 || HDP == 64 || HDP == 80, "head tiles are 32, 64 or 80 columns wide");
  static constexpr int HA = HDP == 80 ? 64 : HDP;  // columns of the first atom
  static constexpr int HB = HDP - HA;              // columns of the second atom (0 or 16)
  static constexpr uint32_t SWZ_A = HA == 64 ? SWZ_128B : SWZ_64B;
  static constexpr uint32_t ROW_A = HA * 2;        // bytes per row of the first atom
  static constexpr uint32_t ROW_B = 32;            // bytes per row of the second atom
  static constexpr int KSTEPS = HDP / 16;

  // byte offset of the second atom in a tile of `rows` rows
  __host__ __device__ static constexpr uint32_t b_off(int rows) { return rows * ROW_A; }

  // K-major descriptor of rows [r0, r0 + 64) for K step k (head columns [16k, 16k + 16)) of a tile of `rows` rows
  __device__ __forceinline__ static uint64_t kdesc(uint32_t tile, int rows, int r0, int k) {
    if (HB > 0 && k == HA / 16) return make_smem_desc(tile + b_off(rows) + r0 * ROW_B, 16, 8 * ROW_B, SWZ_32B);
    return make_smem_desc(tile + r0 * ROW_A + k * 32, 16, 8 * ROW_A, SWZ_A);
  }
  // MN-major descriptors (B operand, N = head columns) of tile rows [16ks, 16ks + 16): first and second atom
  __device__ __forceinline__ static uint64_t ndesc_a(uint32_t tile, int ks) {
    return make_smem_desc(tile + ks * 16 * ROW_A, 0, 8 * ROW_A, SWZ_A);
  }
  __device__ __forceinline__ static uint64_t ndesc_b(uint32_t tile, int rows, int ks) {
    return make_smem_desc(tile + b_off(rows) + ks * 16 * ROW_B, 0, 8 * ROW_B, SWZ_32B);
  }

  // TMA loads of one box (matrix rows [row, row + box rows), columns [col, col + HDP)) into tile rows [r0, ...)
  __device__ __forceinline__ static void load(uint8_t* tile, int rows, int r0, const CUtensorMap* ma,
                                              const CUtensorMap* mb, uint64_t* bar, int col, int row) {
    tma_load_2d(tile + r0 * ROW_A, ma, bar, col, row);
    if (HB > 0) tma_load_2d(tile + b_off(rows) + r0 * ROW_B, mb, bar, col + HA, row);
  }
};

// D[128 x HDP] (+)= sum_k A_k B_k with B a head tile of `rows` rows read MN-major (N = the head columns): one
// wg_mma_128 per atom, the second into columns [64, 80) of buf
template <int HDP, int TA, int KSTEPS, class FA>
__device__ __forceinline__ void wg_mma_128_head(float* buf, int ld, FA adesc, uint32_t btile, int rows, bool accumulate) {
  using HT = HeadTile<HDP>;
  wg_mma_128<HT::HA, TA, 1, KSTEPS>(buf, ld, adesc, [&](int ks) { return HT::ndesc_a(btile, ks); }, accumulate);
  if constexpr (HT::HB > 0)
    wg_mma_128<HT::HB, TA, 1, KSTEPS>(buf + HT::HA, ld, adesc, [&](int ks) { return HT::ndesc_b(btile, rows, ks); },
                                      accumulate);
}

// NCOL fp32 values of an accumulator row, times mul, as fp16 at dst (16-byte stores)
template <int NCOL>
__device__ __forceinline__ void store_row_f16(const float* src, float mul, __half* dst) {
#pragma unroll
  for (int c0 = 0; c0 < NCOL; c0 += 16) {
    uint32_t raw[16];
    ld_row16(src + c0, raw);
    uint32_t o[8];
#pragma unroll
    for (int u = 0; u < 8; ++u) {
      const __half2 h = __floats2half2_rn(__uint_as_float(raw[2 * u]) * mul, __uint_as_float(raw[2 * u + 1]) * mul);
      o[u] = *reinterpret_cast<const uint32_t*>(&h);
    }
    *reinterpret_cast<uint4*>(dst + c0) = make_uint4(o[0], o[1], o[2], o[3]);
    *reinterpret_cast<uint4*>(dst + c0 + 8) = make_uint4(o[4], o[5], o[6], o[7]);
  }
}

// The tensor maps of a [rows, cols] fp16 matrix that head tiles of padded width hdp load from, with box_rows-row
// boxes: ma covers the first atom's columns, mb the second's (a copy of ma when the tile has one atom)
inline int head_tile_tmaps(CUtensorMap* ma, CUtensorMap* mb, const void* base, uint64_t cols, uint64_t rows,
                           int64_t ld, int hdp, int box_rows) {
  const uint64_t dims[2] = {cols, rows};
  const uint64_t strides[1] = {(uint64_t)ld * 2};
  const uint32_t ha = hdp == 80 ? 64 : (uint32_t)hdp;
  const uint32_t box[2] = {ha, (uint32_t)box_rows};
  int rc = cached_tmap_16bit(ma, base, 2, dims, strides, box,
                             ha == 64 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_64B);
  if (rc || hdp != 80) {
    *mb = *ma;
    return rc;
  }
  const uint32_t box_b[2] = {16, (uint32_t)box_rows};
  return cached_tmap_16bit(mb, base, 2, dims, strides, box_b, CU_TENSOR_MAP_SWIZZLE_32B);
}

}  // namespace fvit
