// HBM-bound kernels of the FasterViT forward path (everything that is not a GEMM): weight packing,
// BN/layer-scale folding, the 3->C stem convolution, LayerNorm (+ positional-embedding add, gather),
// carrier-token initialiser, positional MLPs / attention-bias table, carrier->window propagation,
// head pooling. All are coalesced along the channel dimension (NHWC / token-major rows) with
// vectorised 16-byte accesses where the shape allows. Contracts are in include/fvit.h.
#include <cuda_fp16.h>

#include <cstdlib>

#include "../../include/fvit.h"
#include "common.h"

namespace fvit {

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// ------------------------------------------------------------------------------ weight packing
// dst[r][c] (fp16, row stride ldd, zero padded to `cols_pad`) = src[r][c] (fp32, row stride lds)
__global__ void cast_pad_kernel(const float* __restrict__ src, long long lds, __half* __restrict__ dst,
                                long long ldd, int rows, int cols, int cols_pad) {
  const long long total = (long long)rows * cols_pad;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int r = (int)(i / cols_pad), c = (int)(i % cols_pad);
    dst[r * ldd + c] = __float2half_rn(c < cols ? src[r * lds + c] : 0.f);
  }
}

// conv weight [Cout][Cin][3][3] fp32 -> [Cout][9][kc_pad] fp16 (tap-major, channel innermost)
// transpose_io != 0 builds the data-gradient operand [Cin][9 (flipped)][co_pad] instead.
__global__ void pack_conv3x3_kernel(const float* __restrict__ w, __half* __restrict__ dst, int cout,
                                    int cin, int kc_pad, int transpose_io) {
  const int rows = transpose_io ? cin : cout;
  const int inner = transpose_io ? cout : cin;
  const long long total = (long long)rows * 9 * kc_pad;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % kc_pad);
    const int tap = (int)((i / kc_pad) % 9);
    const int r = (int)(i / ((long long)kc_pad * 9));
    float v = 0.f;
    if (c < inner) {
      if (!transpose_io)
        v = w[((long long)r * cin + c) * 9 + tap];
      else
        v = w[((long long)c * cin + r) * 9 + (8 - tap)];
    }
    dst[i] = __float2half_rn(v);
  }
}

// Explicit-tap variant: dst[r][j][c] for j < ntaps uses source tap taps[j] (no flip):
//   transpose_io == 0: dst[co][j][ci] = w[co][ci][taps[j]] ; != 0: dst[ci][j][co] = w[co][ci][taps[j]]
struct TapList { int t[9]; };
__global__ void pack_conv3x3_taps_kernel(const float* __restrict__ w, __half* __restrict__ dst, int cout, int cin,
                                         int kc_pad, int transpose_io, int ntaps, TapList taps) {
  const int rows = transpose_io ? cin : cout;
  const int inner = transpose_io ? cout : cin;
  const long long total = (long long)rows * ntaps * kc_pad;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % kc_pad);
    const int j = (int)((i / kc_pad) % ntaps);
    const int r = (int)(i / ((long long)kc_pad * ntaps));
    float v = 0.f;
    if (c < inner) v = transpose_io ? w[((long long)c * cin + r) * 9 + taps.t[j]] : w[((long long)r * cin + c) * 9 + taps.t[j]];
    dst[i] = __float2half_rn(v);
  }
}

// Head-padded packing for the tensor-core attention path: blocks of `hd` rows (pad_rows) and/or
// columns (pad_cols) of the fp32 source are spread to blocks of `hdp` >= hd with zero fill, e.g. the
// qkv weight [3*h*hd, C] -> [3*h*hdp, C] and the proj weight [C, h*hd] -> [C, h*hdp].
__global__ void cast_headpad_kernel(const float* __restrict__ src, long long lds, __half* __restrict__ dst,
                                    long long ldd, int rows_dst, int cols_dst, int hd, int hdp,
                                    int pad_rows, int pad_cols) {
  const long long total = (long long)rows_dst * cols_dst;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int r = (int)(i / cols_dst), c = (int)(i % cols_dst);
    int sr = r, sc = c;
    bool ok = true;
    if (pad_rows) {
      const int d = r % hdp;
      ok = ok && d < hd;
      sr = (r / hdp) * hd + d;
    }
    if (pad_cols) {
      const int d = c % hdp;
      ok = ok && d < hd;
      sc = (c / hdp) * hd + d;
    }
    dst[r * ldd + c] = __float2half_rn(ok ? src[sr * lds + sc] : 0.f);
  }
}

// 8 elements per thread (two 16-byte loads, one 16-byte store) for the common aligned case
__global__ void __launch_bounds__(256)
cast_pad_vec8_kernel(const float* __restrict__ src, long long lds, __half* __restrict__ dst, long long ldd, int rows,
                     int cols, int cols_pad) {
  const unsigned nv = (unsigned)cols_pad >> 3;
  const unsigned total = (unsigned)rows * nv;
  for (unsigned i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    const unsigned r = i / nv, c = (i - r * nv) << 3;
    float v[8];
    if (c + 8 <= (unsigned)cols) {
      const float4 a = *reinterpret_cast<const float4*>(src + (long long)r * lds + c);
      const float4 b = *reinterpret_cast<const float4*>(src + (long long)r * lds + c + 4);
      v[0] = a.x, v[1] = a.y, v[2] = a.z, v[3] = a.w, v[4] = b.x, v[5] = b.y, v[6] = b.z, v[7] = b.w;
    } else {
#pragma unroll
      for (int k = 0; k < 8; ++k) v[k] = c + k < (unsigned)cols ? src[(long long)r * lds + c + k] : 0.f;
    }
    uint4 o;
    uint32_t* ow = reinterpret_cast<uint32_t*>(&o);
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const __half2 h = __floats2half2_rn(v[2 * k], v[2 * k + 1]);
      ow[k] = *reinterpret_cast<const uint32_t*>(&h);
    }
    *reinterpret_cast<uint4*>(dst + (long long)r * ldd + c) = o;
  }
}
__global__ void __launch_bounds__(256)
cast_headpad_vec8_kernel(const float* __restrict__ src, long long lds, __half* __restrict__ dst, long long ldd,
                         int rows_dst, int cols_dst, int hd, int hdp, int pad_rows, int pad_cols) {
  const unsigned nv = (unsigned)cols_dst >> 3;
  const unsigned total = (unsigned)rows_dst * nv;
  for (unsigned i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    const unsigned r = i / nv, c = (i - r * nv) << 3;
    bool row_ok = true;
    unsigned sr = r;
    if (pad_rows) {
      const unsigned d = r % (unsigned)hdp;
      row_ok = d < (unsigned)hd;
      sr = (r / (unsigned)hdp) * hd + d;
    }
    float v[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) v[k] = 0.f;
    if (row_ok) {
      if (!pad_cols) {
        const float4 a = *reinterpret_cast<const float4*>(src + (long long)sr * lds + c);
        const float4 b = *reinterpret_cast<const float4*>(src + (long long)sr * lds + c + 4);
        v[0] = a.x, v[1] = a.y, v[2] = a.z, v[3] = a.w, v[4] = b.x, v[5] = b.y, v[6] = b.z, v[7] = b.w;
      } else {
        // 8 destination columns lie inside one padded head (hdp % 8 == 0): d .. d+7 of head c / hdp
        const unsigned d0 = c % (unsigned)hdp, sc0 = (c / (unsigned)hdp) * hd + d0;
#pragma unroll
        for (int k = 0; k < 8; ++k)
          if (d0 + k < (unsigned)hd) v[k] = src[(long long)sr * lds + sc0 + k];
      }
    }
    uint4 o;
    uint32_t* ow = reinterpret_cast<uint32_t*>(&o);
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const __half2 h = __floats2half2_rn(v[2 * k], v[2 * k + 1]);
      ow[k] = *reinterpret_cast<const uint32_t*>(&h);
    }
    *reinterpret_cast<uint4*>(dst + (long long)r * ldd + c) = o;
  }
}
__global__ void vec_headpad_kernel(const float* __restrict__ src, float* __restrict__ dst, int n_dst, int hd,
                                   int hdp) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_dst) return;
  const int d = i % hdp;
  dst[i] = d < hd ? src[(i / hdp) * hd + d] : 0.f;
}

// Per-channel epilogue vectors:  s = bn ? w*rsqrt(var+eps) : 1 ; t = bn ? b - mean*s : 0 ;
// t += bias*s ; then both *= layer_scale (if given).  y = acc*s + t reproduces
// layer_scale * BN(acc + bias) (fv.py:504-510) or layer_scale * (acc + bias) (fv.py:690-691).
__global__ void affine_fold_kernel(float* __restrict__ scale, float* __restrict__ shift, int n,
                                   const float* bn_w, const float* bn_b, const float* bn_mean,
                                   const float* bn_var, float eps, const float* bias,
                                   const float* ls) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  float s = 1.f, t = 0.f;
  if (bn_w) {
    s = bn_w[i] * rsqrtf(bn_var[i] + eps);
    t = bn_b[i] - bn_mean[i] * s;
  }
  if (bias) t += bias[i] * s;
  if (ls) {
    s *= ls[i];
    t *= ls[i];
  }
  scale[i] = s;
  shift[i] = t;
}

// ------------------------------------------------------------------------------ stem conv 3x3 s2
// x fp32 [B,3,H,W] (arbitrary strides) -> y = relu(conv(x) * scale + shift) as fp16 rows of `cout`
// channels written at out_row_map[b*Ho*Wo + oh*Wo + ow] (the parity-plane layout conv2 consumes).
// One thread per (pixel, 16 output channels): the 27 taps sit in registers, weights are read from
// shared memory as [27][cout] float4 broadcasts (one LDS.128 per 4 FMAs), and the cout/16 threads
// of a pixel write one contiguous 2*cout-byte row. fp32 math (K = 27 is too thin for tensor cores;
// the kernel is HBM/LSU bound: 3*H*W*4 B in, cout*H*W/2 B out per image).
template <int CIN>
__global__ void __launch_bounds__(256)
    stem_conv_kernel(const float* __restrict__ x, long long sb, long long sc, long long sh, long long sw,
                     int B, int H, int W, const float* __restrict__ wgt, int cout,
                     const float* __restrict__ scale, const float* __restrict__ shift, int relu,
                     const int* __restrict__ out_row_map, __half* __restrict__ out, long long ldo,
                     float* __restrict__ col_sum, float* __restrict__ col_sumsq) {
  extern __shared__ float sw_[];  // [CIN*9][cout] then (statistics) [2][cout]
  constexpr int K = CIN * 9;
  for (int i = threadIdx.x; i < cout * K; i += blockDim.x) {
    const int co = i / K, k = i % K;
    sw_[k * cout + co] = wgt[i];
  }
  float* red = sw_ + K * cout;
  if (col_sum)
    for (int i = threadIdx.x; i < 2 * cout; i += blockDim.x) red[i] = 0.f;
  __syncthreads();
  const int Ho = (H + 1) / 2, Wo = (W + 1) / 2;
  const int groups = cout / 16;
  const long long total = (long long)B * Ho * Wo * groups;
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  const bool active = i < total;
  float acc[16];
#pragma unroll
  for (int j = 0; j < 16; ++j) acc[j] = 0.f;
  int g = 0;
  long long pix = 0;
  if (active) {
    g = (int)(i % groups);
    pix = i / groups;
    const int ow = (int)(pix % Wo);
    const int oh = (int)((pix / Wo) % Ho);
    const int b = (int)(pix / ((long long)Wo * Ho));
    float in[K];
#pragma unroll
    for (int c = 0; c < CIN; ++c)
#pragma unroll
      for (int r = 0; r < 3; ++r)
#pragma unroll
        for (int s = 0; s < 3; ++s) {
          const int ih = 2 * oh + r - 1, iw = 2 * ow + s - 1;
          in[c * 9 + r * 3 + s] =
              (ih >= 0 && ih < H && iw >= 0 && iw < W) ? __ldg(x + b * sb + c * sc + ih * sh + iw * sw) : 0.f;
        }
#pragma unroll
    for (int k = 0; k < K; ++k) {
      const float4* wr = reinterpret_cast<const float4*>(sw_ + k * cout + g * 16);
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const float4 w4 = wr[q];
        acc[4 * q + 0] = fmaf(in[k], w4.x, acc[4 * q + 0]);
        acc[4 * q + 1] = fmaf(in[k], w4.y, acc[4 * q + 1]);
        acc[4 * q + 2] = fmaf(in[k], w4.z, acc[4 * q + 2]);
        acc[4 * q + 3] = fmaf(in[k], w4.w, acc[4 * q + 3]);
      }
    }
  }
  if (col_sum) {
    // train-mode BatchNorm statistics of the raw conv output: block-level reduction, then atomics
    if (active) {
#pragma unroll
      for (int j = 0; j < 16; ++j) {
        atomicAdd(&red[g * 16 + j], acc[j]);
        atomicAdd(&red[cout + g * 16 + j], acc[j] * acc[j]);
      }
    }
    __syncthreads();
    for (int j = threadIdx.x; j < cout; j += blockDim.x) {
      atomicAdd(col_sum + j, red[j]);
      atomicAdd(col_sumsq + j, red[cout + j]);
    }
  }
  if (active && out) {
    const int orow = out_row_map ? out_row_map[pix] : (int)pix;
    if (orow >= 0) {
      uint32_t pk[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        float v0 = acc[2 * j], v1 = acc[2 * j + 1];
        if (scale) {
          v0 = fmaf(v0, __ldg(scale + g * 16 + 2 * j), __ldg(shift + g * 16 + 2 * j));
          v1 = fmaf(v1, __ldg(scale + g * 16 + 2 * j + 1), __ldg(shift + g * 16 + 2 * j + 1));
        }
        if (relu) {
          v0 = fmaxf(v0, 0.f);
          v1 = fmaxf(v1, 0.f);
        }
        const __half2 h = __floats2half2_rn(v0, v1);
        pk[j] = *reinterpret_cast<const uint32_t*>(&h);
      }
      uint4* o = reinterpret_cast<uint4*>(out + (long long)orow * ldo + g * 16);
      o[0] = make_uint4(pk[0], pk[1], pk[2], pk[3]);
      o[1] = make_uint4(pk[4], pk[5], pk[6], pk[7]);
    }
  }
}

// im2col of the 3x3 / stride-2 / pad-1 stem convolution: out[pixel][c*9 + r*3 + s] = (half)x[b][c][2oh+r-1][2ow+s-1]
// (zero outside the image, zero in columns >= 9*CIN). One thread per output pixel writes one `ldo`-wide
// fp16 row with 16-byte stores; the GEMM kernel then runs the 27-deep contraction on tensor cores.
template <int CIN>
__global__ void __launch_bounds__(256)
    stem_im2col_kernel(const float* __restrict__ x, long long sb, long long sc, long long sh, long long sw,
                       int B, int H, int W, __half* __restrict__ out, int ldo) {
  const int Ho = (H + 1) / 2, Wo = (W + 1) / 2;
  const unsigned total = (unsigned)B * Ho * Wo;
  const unsigned pix = blockIdx.x * blockDim.x + threadIdx.x;
  if (pix >= total) return;
  const int ow = pix % Wo;
  const int oh = (pix / Wo) % Ho;
  const int b = pix / ((unsigned)Wo * Ho);
  constexpr int K = CIN * 9;
  constexpr int KP = (K + 7) / 8 * 8;
  __half v[KP];
#pragma unroll
  for (int c = 0; c < CIN; ++c)
#pragma unroll
    for (int r = 0; r < 3; ++r)
#pragma unroll
      for (int s = 0; s < 3; ++s) {
        const int ih = 2 * oh + r - 1, iw = 2 * ow + s - 1;
        const float f = (ih >= 0 && ih < H && iw >= 0 && iw < W) ? __ldg(x + b * sb + c * sc + ih * sh + iw * sw) : 0.f;
        v[c * 9 + r * 3 + s] = __float2half_rn(f);
      }
#pragma unroll
  for (int k = K; k < KP; ++k) v[k] = __float2half_rn(0.f);
  uint4* o = reinterpret_cast<uint4*>(out + (long long)pix * ldo);
#pragma unroll
  for (int q = 0; q < KP / 8; ++q) o[q] = *reinterpret_cast<const uint4*>(&v[q * 8]);
  for (int q = KP / 8; q < ldo / 8; ++q) o[q] = make_uint4(0, 0, 0, 0);
}

// The same im2col for any channel count (in_chans != 3): one thread per (pixel, 8-column group), so a thread holds
// 8 taps whatever cin is. Consecutive threads write consecutive 16-byte pieces of the (contiguous) output rows.
__global__ void __launch_bounds__(256)
    stem_im2col_any_kernel(const float* __restrict__ x, long long sb, long long sc, long long sh, long long sw,
                           int B, int cin, int H, int W, __half* __restrict__ out, int ldo) {
  const int Ho = (H + 1) / 2, Wo = (W + 1) / 2;
  const int groups = ldo / 8, K = cin * 9;
  const long long total = (long long)B * Ho * Wo * groups;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int q = (int)(i % groups);
    const long long pix = i / groups;
    const int ow = (int)(pix % Wo);
    const int oh = (int)((pix / Wo) % Ho);
    const int b = (int)(pix / ((long long)Wo * Ho));
    __align__(16) __half v[8];
#pragma unroll
    for (int u = 0; u < 8; ++u) {
      const int k = q * 8 + u;
      float f = 0.f;
      if (k < K) {
        const int c = k / 9, t = k - c * 9;
        const int ih = 2 * oh + t / 3 - 1, iw = 2 * ow + t % 3 - 1;
        if (ih >= 0 && ih < H && iw >= 0 && iw < W) f = __ldg(x + b * sb + c * sc + ih * sh + iw * sw);
      }
      v[u] = __float2half_rn(f);
    }
    *reinterpret_cast<uint4*>(out + pix * ldo + q * 8) = *reinterpret_cast<const uint4*>(v);
  }
}

// ------------------------------------------------------------------------------ LayerNorm forward
// One warp per row. v = x[in_map ? in_map[r] : r] (+ add[(r % group) - skip] if (r % group) >= skip);
// optionally written back as fp32 to wb[r]; y = (v - mean) * rstd * gamma + beta written as fp16 to
// out[out_map ? out_map[r] : r]. Two-pass statistics in registers (biased variance, like
// F.layer_norm). Saves mean / rstd when requested (backward).
// LPR lanes cooperate on one row (32 / LPR rows per warp), each lane holding up to MAXV float4.
template <int LPR, int MAXV>
__global__ void __launch_bounds__(256)
    ln_fwd_kernel(const float* __restrict__ x, long long ldx, const int* __restrict__ in_map, int rows,
                  int C, const float* __restrict__ add, int group, int skip, float* __restrict__ wb,
                  long long ldwb, const float* __restrict__ gamma, const float* __restrict__ beta,
                  float eps, __half* __restrict__ out, long long ldo, const int* __restrict__ out_map,
                  float* __restrict__ mean_out, float* __restrict__ rstd_out, __half* __restrict__ xhat_out,
                  long long ldxh) {
  constexpr int RPW = 32 / LPR;  // rows per warp
  const int lane = threadIdx.x & 31;
  const int sl = lane % LPR;     // lane within the row group
  const int nvec = C >> 2;
  const long long warp_global = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const long long r = warp_global * RPW + lane / LPR;
  const bool active = r < rows;
  float4 v[MAXV];
  float s = 0.f;
  if (active) {
    const long long src = in_map ? in_map[r] : r;
    const float4* xr = reinterpret_cast<const float4*>(x + src * ldx);
    const float4* ar = nullptr;
    if (add) {
      const int t = (int)(r % group);
      if (t >= skip) ar = reinterpret_cast<const float4*>(add + (long long)(t - skip) * C);
    }
#pragma unroll
    for (int j = 0; j < MAXV; ++j) {
      const int i = sl + LPR * j;
      if (i < nvec) {
        float4 t4 = xr[i];
        if (ar) {
          const float4 a4 = ar[i];
          t4.x += a4.x, t4.y += a4.y, t4.z += a4.z, t4.w += a4.w;
        }
        v[j] = t4;
        s += t4.x + t4.y + t4.z + t4.w;
      }
    }
  }
#pragma unroll
  for (int o = LPR / 2; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  const float mean = s / C;
  float q = 0.f;
  if (active) {
#pragma unroll
    for (int j = 0; j < MAXV; ++j) {
      const int i = sl + LPR * j;
      if (i < nvec) {
        const float a = v[j].x - mean, b = v[j].y - mean, c = v[j].z - mean, d = v[j].w - mean;
        q += a * a + b * b + c * c + d * d;
      }
    }
  }
#pragma unroll
  for (int o = LPR / 2; o > 0; o >>= 1) q += __shfl_xor_sync(0xffffffffu, q, o);
  if (!active) return;
  const float rstd = rsqrtf(q / C + eps);
  if (wb) {
    float4* wr = reinterpret_cast<float4*>(wb + r * ldwb);
#pragma unroll
    for (int j = 0; j < MAXV; ++j) {
      const int i = sl + LPR * j;
      if (i < nvec) wr[i] = v[j];
    }
  }
  if (mean_out && sl == 0) {
    mean_out[r] = mean;
    rstd_out[r] = rstd;
  }
  if (xhat_out) {  // normalised (pre-affine) value, saved for the backward pass
    __half* o = xhat_out + r * ldxh;
#pragma unroll
    for (int j = 0; j < MAXV; ++j) {
      const int i = sl + LPR * j;
      if (i < nvec) {
        const __half2 h0 = __floats2half2_rn((v[j].x - mean) * rstd, (v[j].y - mean) * rstd);
        const __half2 h1 = __floats2half2_rn((v[j].z - mean) * rstd, (v[j].w - mean) * rstd);
        uint2 pk;
        pk.x = *reinterpret_cast<const uint32_t*>(&h0);
        pk.y = *reinterpret_cast<const uint32_t*>(&h1);
        *reinterpret_cast<uint2*>(o + 4 * i) = pk;
      }
    }
  }
  const long long orow = out_map ? out_map[r] : r;
  if (orow >= 0) {
    __half* o = out + orow * ldo;
    const float4* g4 = reinterpret_cast<const float4*>(gamma);
    const float4* b4 = reinterpret_cast<const float4*>(beta);
#pragma unroll
    for (int j = 0; j < MAXV; ++j) {
      const int i = sl + LPR * j;
      if (i < nvec) {
        const float4 g = __ldg(g4 + i), b = __ldg(b4 + i);
        const __half2 h0 = __floats2half2_rn((v[j].x - mean) * rstd * g.x + b.x,
                                             (v[j].y - mean) * rstd * g.y + b.y);
        const __half2 h1 = __floats2half2_rn((v[j].z - mean) * rstd * g.z + b.z,
                                             (v[j].w - mean) * rstd * g.w + b.w);
        uint2 pk;
        pk.x = *reinterpret_cast<const uint32_t*>(&h0);
        pk.y = *reinterpret_cast<const uint32_t*>(&h1);
        *reinterpret_cast<uint2*>(o + 4 * i) = pk;
      }
    }
  }
}

// ------------------------------------------------------------------------------ attention core (SIMT)
// One CTA per (group of S tokens, head): P = softmax(q k^T * scale + bias[h]) ; out = P v.
// qkv fp16 [rows, 3C] (q | k | v, head-major inside each), out fp16 [rows, C]. fp32 math throughout.
// Generic in S and head_dim; serves the shapes the tensor-core attention kernels do not cover
// (head dims above 64, windows the key-loop kernel cannot stage).
__global__ void attn_core_simt_kernel(const __half* __restrict__ qkv, long long ldq, int S, int hd,
                                      int heads, int C, const float* __restrict__ bias, float scale,
                                      __half* __restrict__ out, long long ldo,
                                      float* __restrict__ probs_out) {
  extern __shared__ float sm[];
  const int hdp = hd + 1;
  float* sq = sm;                 // [S][hd+1]
  float* sk = sq + S * hdp;       // [S][hd+1]
  float* sv = sk + S * hdp;       // [S][hd+1]
  float* sp = sv + S * hdp;       // [S][S+1]
  const int g = blockIdx.x / heads, h = blockIdx.x % heads;
  const long long row0 = (long long)g * S;
  for (int i = threadIdx.x; i < S * hd; i += blockDim.x) {
    const int t = i / hd, d = i % hd;
    const __half* base = qkv + (row0 + t) * ldq + h * hd + d;
    sq[t * hdp + d] = __half2float(base[0]) * scale;
    sk[t * hdp + d] = __half2float(base[C]);
    sv[t * hdp + d] = __half2float(base[2 * C]);
  }
  __syncthreads();
  const float* bh = bias ? bias + (long long)h * S * S : nullptr;
  for (int i = threadIdx.x; i < S * S; i += blockDim.x) {
    const int r = i / S, c = i % S;
    float a = 0.f;
    for (int d = 0; d < hd; ++d) a = fmaf(sq[r * hdp + d], sk[c * hdp + d], a);
    sp[r * (S + 1) + c] = a + (bh ? bh[i] : 0.f);
  }
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nwarps = blockDim.x >> 5;
  for (int r = warp; r < S; r += nwarps) {
    float* pr = sp + r * (S + 1);
    float m = -INFINITY;
    for (int c = lane; c < S; c += 32) m = fmaxf(m, pr[c]);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    float s = 0.f;
    for (int c = lane; c < S; c += 32) {
      const float e = __expf(pr[c] - m);
      pr[c] = e;
      s += e;
    }
    s = warp_sum(s);
    const float inv = 1.f / s;
    for (int c = lane; c < S; c += 32) pr[c] *= inv;
  }
  __syncthreads();
  if (probs_out) {
    float* po = probs_out + ((long long)g * heads + h) * S * S;
    for (int i = threadIdx.x; i < S * S; i += blockDim.x) po[i] = sp[(i / S) * (S + 1) + (i % S)];
  }
  for (int i = threadIdx.x; i < S * hd; i += blockDim.x) {
    const int r = i / hd, d = i % hd;
    float a = 0.f;
    for (int c = 0; c < S; ++c) a = fmaf(sp[r * (S + 1) + c], sv[c * hdp + d], a);
    out[(row0 + r) * ldo + h * hd + d] = __float2half_rn(a);
  }
}

// Streaming variant for windows whose score matrix does not fit in shared memory (the 21k fine-tuned
// FasterViT-4 models: window 14 / 24 / 32 / 48 -> S = 196 .. 2304, fv.py:1253-1418): one CTA per (64-query
// tile, group, head) walks the keys in tiles of 64 with the running max / running sum recurrence
//   m' = max(m, rowmax(s)) ; l' = l e^(m-m') + sum e^(s-m') ; O' = O e^(m-m') + e^(s-m') V ,
// so only a 64 x 64 score tile is ever resident. Same operand layout and fp32 math as attn_core_simt_kernel.
constexpr int ATT_QT = 64, ATT_KT = 64;
__global__ void __launch_bounds__(256)
attn_stream_simt_kernel(const __half* __restrict__ qkv, long long ldq, int S, int hd, int heads, int C,
                        const float* __restrict__ bias, float scale, __half* __restrict__ out, long long ldo) {
  extern __shared__ float sm[];
  const int hdp = hd + 1;
  float* sq = sm;                          // [QT][hd+1]  (pre-scaled queries)
  float* sk = sq + ATT_QT * hdp;           // [KT][hd+1]
  float* sv = sk + ATT_KT * hdp;           // [KT][hd+1]
  float* so = sv + ATT_KT * hdp;           // [QT][hd+1]  running output
  float* ss = so + ATT_QT * hdp;           // [QT][KT+1]  scores -> un-normalised probabilities
  float* sm_ = ss + ATT_QT * (ATT_KT + 1); // [QT] running max
  float* sl = sm_ + ATT_QT;                // [QT] running sum
  float* sa = sl + ATT_QT;                 // [QT] rescale factor of this step
  const int g = blockIdx.y / heads, h = blockIdx.y % heads;
  const int q0 = blockIdx.x * ATT_QT;
  const long long row0 = (long long)g * S;
  const int nq = min(ATT_QT, S - q0);
  for (int i = threadIdx.x; i < ATT_QT * hd; i += blockDim.x) {
    const int t = i / hd, d = i % hd;
    sq[t * hdp + d] = t < nq ? __half2float(qkv[(row0 + q0 + t) * ldq + h * hd + d]) * scale : 0.f;
    so[t * hdp + d] = 0.f;
  }
  for (int i = threadIdx.x; i < ATT_QT; i += blockDim.x) {
    sm_[i] = -INFINITY;
    sl[i] = 0.f;
  }
  const float* bh = bias ? bias + (long long)h * S * S : nullptr;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nwarps = blockDim.x >> 5;
  for (int k0 = 0; k0 < S; k0 += ATT_KT) {
    const int nk = min(ATT_KT, S - k0);
    __syncthreads();  // previous tile fully consumed (and the prologue stores are visible)
    for (int i = threadIdx.x; i < ATT_KT * hd; i += blockDim.x) {
      const int t = i / hd, d = i % hd;
      float kv = 0.f, vv = 0.f;
      if (t < nk) {
        const __half* base = qkv + (row0 + k0 + t) * ldq + h * hd + d;
        kv = __half2float(base[C]);
        vv = __half2float(base[2 * C]);
      }
      sk[t * hdp + d] = kv;
      sv[t * hdp + d] = vv;
    }
    __syncthreads();
    for (int i = threadIdx.x; i < ATT_QT * ATT_KT; i += blockDim.x) {
      const int r = i / ATT_KT, c = i % ATT_KT;
      float a = -INFINITY;
      if (r < nq && c < nk) {
        a = 0.f;
        for (int d = 0; d < hd; ++d) a = fmaf(sq[r * hdp + d], sk[c * hdp + d], a);
        if (bh) a += bh[(long long)(q0 + r) * S + k0 + c];
      }
      ss[r * (ATT_KT + 1) + c] = a;
    }
    __syncthreads();
    for (int r = warp; r < nq; r += nwarps) {
      float* pr = ss + r * (ATT_KT + 1);
      float m = fmaxf(pr[lane], pr[lane + 32]);
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
      const float m_old = sm_[r];
      const float m_new = fmaxf(m_old, m);   // finite: every key tile holds at least one valid key
      const float e0 = __expf(pr[lane] - m_new), e1 = __expf(pr[lane + 32] - m_new);  // exp(-inf) = 0 for masked keys
      pr[lane] = e0;
      pr[lane + 32] = e1;
      const float sum = warp_sum(e0 + e1);
      if (lane == 0) {
        const float alpha = __expf(m_old - m_new);  // 0 on the first tile (m_old = -inf)
        sa[r] = alpha;
        sl[r] = sl[r] * alpha + sum;
        sm_[r] = m_new;
      }
    }
    __syncthreads();
    for (int i = threadIdx.x; i < nq * hd; i += blockDim.x) {
      const int r = i / hd, d = i % hd;
      const float* pr = ss + r * (ATT_KT + 1);
      float a = so[r * hdp + d] * sa[r];
      for (int c = 0; c < nk; ++c) a = fmaf(pr[c], sv[c * hdp + d], a);
      so[r * hdp + d] = a;
    }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < nq * hd; i += blockDim.x) {
    const int r = i / hd, d = i % hd;
    out[(row0 + q0 + r) * ldo + h * hd + d] = __float2half_rn(so[r * hdp + d] / sl[r]);
  }
}

// ------------------------------------------------------------------------------ positional MLPs
// out[p][d] = sum_j relu(w0[j][0]*c[p][0] + w0[j][1]*c[p][1] + b0[j]) * w1[d][j]   (hidden = 512)
// (cpb_mlp of PosEmbMLPSwinv1D / PosEmbMLPSwinv2D, fv.py:223-225, 322-324). One CTA per point p;
// hidden activations in shared memory; one warp per output channel, lanes stride the hidden dim.
__global__ void cpb_mlp_kernel(const float* __restrict__ coords, int P, const float* __restrict__ w0,
                               const float* __restrict__ b0, const float* __restrict__ w1, int D,
                               float* __restrict__ out, float* __restrict__ hidden_out) {
  __shared__ float hid[512];
  const int p = blockIdx.x;
  const float c0 = coords[2 * p], c1 = coords[2 * p + 1];
  for (int j = threadIdx.x; j < 512; j += blockDim.x) {
    const float hv = fmaxf(fmaf(w0[2 * j], c0, fmaf(w0[2 * j + 1], c1, b0[j])), 0.f);
    hid[j] = hv;
    if (hidden_out) hidden_out[(long long)p * 512 + j] = hv;
  }
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nwarps = blockDim.x >> 5;
  for (int d = warp; d < D; d += nwarps) {
    const float* wr = w1 + (long long)d * 512;
    float a = 0.f;
#pragma unroll 4
    for (int j = lane; j < 512; j += 32) a = fmaf(hid[j], wr[j], a);
    a = warp_sum(a);
    if (lane == 0) out[(long long)p * D + d] = a;
  }
}

// Wide-output variant (D >= 64: the additive token embeddings, D = C up to 1568 with only P = 16..169 points).
// One warp per output channel d keeps its w1 row in registers (16 values per lane, j = lane + 32 i) next to the
// matching w0 / b0 entries, re-derives the hidden activations of every point on the fly (3 instructions each)
// and reduces over the lanes; w1 is read exactly once overall instead of once per point. The summation order
// (lane-strided partial sums, then the xor tree) and the hidden formula are those of cpb_mlp_kernel, so the two
// variants agree bit for bit.
__global__ void __launch_bounds__(256)
cpb_mlp_wide_kernel(const float* __restrict__ coords, int P, const float* __restrict__ w0,
                    const float* __restrict__ b0, const float* __restrict__ w1, int D,
                    float* __restrict__ out, float* __restrict__ hidden_out) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (hidden_out) {  // saved for the backward pass: grid-strided so every CTA writes a slice
    const int total = P * 512;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
      const int p = i >> 9, j = i & 511;
      hidden_out[i] = fmaxf(fmaf(__ldg(w0 + 2 * j), __ldg(coords + 2 * p),
                                 fmaf(__ldg(w0 + 2 * j + 1), __ldg(coords + 2 * p + 1), __ldg(b0 + j))), 0.f);
    }
  }
  const int d = blockIdx.x * 8 + warp;
  if (d >= D) return;
  float wa[16], wb[16], bb[16], w1r[16];
  const float* wr = w1 + (long long)d * 512;
#pragma unroll
  for (int i = 0; i < 16; ++i) {
    const int j = lane + 32 * i;
    wa[i] = __ldg(w0 + 2 * j), wb[i] = __ldg(w0 + 2 * j + 1), bb[i] = __ldg(b0 + j), w1r[i] = __ldg(wr + j);
  }
  for (int p = 0; p < P; ++p) {
    const float c0 = __ldg(coords + 2 * p), c1 = __ldg(coords + 2 * p + 1);
    float a = 0.f;
#pragma unroll
    for (int i = 0; i < 16; ++i) a = fmaf(fmaxf(fmaf(wa[i], c0, fmaf(wb[i], c1, bb[i])), 0.f), w1r[i], a);
    a = warp_sum(a);
    if (lane == 0) out[(long long)p * D + d] = a;
  }
}

// bias[h][r][c] = (r >= ng && c >= ng) ? 16*sigmoid(table[index[(r-ng)*L + (c-ng)]][h]) : 0
// with L = ws*ws local tokens and ng = S - L carrier tokens on the top/left (fv.py:276-299). A negative ng (S < L:
// the detection backbone's carrier attention on a grid smaller than the built one) crops the table's top-left instead,
// as F.pad with negative padding does; r, c >= ng then always holds and r - ng < L.
__global__ void attn_bias_kernel(const float* __restrict__ table, const long long* __restrict__ index,
                                 int heads, int S, int L, float* __restrict__ bias) {
  const int ng = S - L;
  const long long total = (long long)heads * S * S;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % S), r = (int)((i / S) % S), h = (int)(i / ((long long)S * S));
    float v = 0.f;
    if (r >= ng && c >= ng) {
      const long long idx = index[(long long)(r - ng) * L + (c - ng)];
      v = 16.f / (1.f + __expf(-table[idx * heads + h]));
    }
    bias[i] = v;
  }
}

// ------------------------------------------------------------------------------ carrier tokens
// TokenInitializer (fv.py:733-738): ct = AvgPool_{kh x kw, stride sh x sw}(dwconv3x3(x) + b), written
// to the carrier rows of the window-major token buffer. x is read through `pix_map` (pixel (b,h,w) of
// the (padded) Hp x Wp map -> row of xs, or -1 for padding pixels which read as zero).
// kNchwTokens (detection backbone, dino/models/dino/fastervit.py:591): the pooled NCHW map of image b is read back as
// [oh*ow, C] tokens without a permute, so value (c, p) lands in token t, channel k with c*oh*ow + p = t*C + k, stored
// to row ct_row_map[b*oh*ow + t]; otherwise value (c, p) is channel c of row ct_row_map[b*oh*ow + p].
template <bool kNchwTokens>
__global__ void token_init_kernel(const float* __restrict__ xs, long long ldx,
                                  const int* __restrict__ pix_map, int B, int Hp, int Wp, int C,
                                  const float* __restrict__ w, const float* __restrict__ bias, int kh,
                                  int kw, int sh, int sw, int oh, int ow,
                                  const int* __restrict__ ct_row_map, float* __restrict__ out,
                                  long long ldo) {
  const long long total = (long long)B * oh * ow * C;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % C);
    const long long pos = i / C;
    const int x0 = (int)(pos % ow), y0 = (int)((pos / ow) % oh), b = (int)(pos / ((long long)ow * oh));
    float wl[9];
#pragma unroll
    for (int t = 0; t < 9; ++t) wl[t] = w[c * 9 + t];
    float acc = 0.f;
    for (int py = 0; py < kh; ++py)
      for (int px = 0; px < kw; ++px) {
        const int cy = y0 * sh + py, cx = x0 * sw + px;
#pragma unroll
        for (int r = 0; r < 3; ++r)
#pragma unroll
          for (int s = 0; s < 3; ++s) {
            const int iy = cy + r - 1, ix = cx + s - 1;
            if (iy >= 0 && iy < Hp && ix >= 0 && ix < Wp) {
              const int row = pix_map[((long long)b * Hp + iy) * Wp + ix];
              if (row >= 0) acc = fmaf(wl[r * 3 + s], xs[(long long)row * ldx + c], acc);
            }
          }
      }
    const float v = acc / (float)(kh * kw) + bias[c];
    if (kNchwTokens) {
      const long long hw = (long long)oh * ow;
      const long long f = (long long)c * hw + (pos - (long long)b * hw);
      out[(long long)ct_row_map[(long long)b * hw + f / C] * ldo + f % C] = v;
    } else {
      out[(long long)ct_row_map[pos] * ldo + c] = v;
    }
  }
}

// Propagation (fv.py:697-700): x[row] += gamma[c] * x[src_map[row]][c] for window-token rows
// (src_map < 0: untouched). gamma == nullptr means 1.
__global__ void propagate_kernel(float* __restrict__ xs, long long ldx, const int* __restrict__ src_map,
                                 int rows, int C, const float* __restrict__ gamma) {
  const int c4 = C >> 2;
  const long long total = (long long)rows * c4;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int j = (int)(i % c4);
    const long long r = i / c4;
    const int src = src_map[r];
    if (src < 0) continue;
    float4 v = reinterpret_cast<float4*>(xs + r * ldx)[j];
    const float4 s = reinterpret_cast<const float4*>(xs + (long long)src * ldx)[j];
    float4 g = make_float4(1.f, 1.f, 1.f, 1.f);
    if (gamma) g = reinterpret_cast<const float4*>(gamma)[j];
    v.x = fmaf(g.x, s.x, v.x), v.y = fmaf(g.y, s.y, v.y), v.z = fmaf(g.z, s.z, v.z),
    v.w = fmaf(g.w, s.w, v.w);
    reinterpret_cast<float4*>(xs + r * ldx)[j] = v;
  }
}

// ------------------------------------------------------------------------------ head
// pooled[b][c] = (mean_t x[row_map(b, t)][c]) * scale[c] + shift[c]  -> fp16  (BatchNorm2d folded
// into the average pool, fv.py:953-958). One thread per (b, 4 channels).
__global__ void pool_affine_kernel(const float* __restrict__ xs, long long ldx,
                                   const int* __restrict__ row_map, int B, int T, int C,
                                   const float* __restrict__ scale, const float* __restrict__ shift,
                                   __half* __restrict__ out, long long ldo) {
  const int c4 = C >> 2;
  const long long total = (long long)B * c4;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int j = (int)(i % c4);
    const int b = (int)(i / c4);
    float4 a = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int t = 0; t < T; ++t) {
      const long long row = row_map ? row_map[(long long)b * T + t] : (long long)b * T + t;
      const float4 v = reinterpret_cast<const float4*>(xs + row * ldx)[j];
      a.x += v.x, a.y += v.y, a.z += v.z, a.w += v.w;
    }
    const float inv = 1.f / T;
    const float4 s = reinterpret_cast<const float4*>(scale)[j];
    const float4 h = reinterpret_cast<const float4*>(shift)[j];
    const __half2 h0 = __floats2half2_rn(a.x * inv * s.x + h.x, a.y * inv * s.y + h.y);
    const __half2 h1 = __floats2half2_rn(a.z * inv * s.z + h.z, a.w * inv * s.w + h.w);
    uint2 pk;
    pk.x = *reinterpret_cast<const uint32_t*>(&h0);
    pk.y = *reinterpret_cast<const uint32_t*>(&h1);
    *reinterpret_cast<uint2*>(out + (long long)b * ldo + 4 * j) = pk;
  }
}

// forward_features (fv.py:949-953): the BatchNorm-ed last-level map in the reference's NCHW layout,
// out[b][c][t] = xs[row_map[b*T + t]][c] * scale[c] + shift[c]; 32 x 32 tiles transposed through shared memory so
// both the token-major reads and the NCHW writes are coalesced.
__global__ void feature_map_kernel(const float* __restrict__ xs, long long ldx, const int* __restrict__ row_map,
                                   int T, int C, const float* __restrict__ scale, const float* __restrict__ shift,
                                   float* __restrict__ out) {
  __shared__ float tile[32][33];
  const int b = blockIdx.z, t0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
  for (int i = threadIdx.y; i < 32; i += 8) {
    const int t = t0 + i, c = c0 + threadIdx.x;
    float v = 0.f;
    if (t < T && c < C) {
      const long long row = row_map ? row_map[(long long)b * T + t] : (long long)b * T + t;
      v = fmaf(xs[row * ldx + c], scale[c], shift[c]);
    }
    tile[i][threadIdx.x] = v;
  }
  __syncthreads();
  for (int i = threadIdx.y; i < 32; i += 8) {
    const int c = c0 + i, t = t0 + threadIdx.x;
    if (t < T && c < C) out[((long long)b * C + c) * T + t] = tile[threadIdx.x][i];
  }
}

// forward_head (fv.py:955-958): AdaptiveAvgPool2d(1) + flatten of an NCHW fp32 map -> fp16 classifier operand;
// one warp per (image, channel).
__global__ void nchw_pool_kernel(const float* __restrict__ x, int BC, int T, int C, __half* __restrict__ out,
                                 long long ldo) {
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (warp >= BC) return;
  const float* src = x + (long long)warp * T;
  float a = 0.f;
  for (int t = lane; t < T; t += 32) a += src[t];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) a += __shfl_xor_sync(0xffffffffu, a, o);
  if (lane == 0) out[(long long)(warp / C) * ldo + warp % C] = __float2half_rn(a / T);
}

static inline int grid_for(long long total, int block) {
  long long g = (total + block - 1) / block;
  const long long cap = (long long)num_sms() * 16;
  if (g > cap) g = cap;
  if (g < 1) g = 1;
  return (int)g;
}

}  // namespace fvit

using namespace fvit;

extern "C" {

int fvit_cast_pad_f16(const float* src, int64_t lds, void* dst, int64_t ldd, int32_t rows,
                      int32_t cols, int32_t cols_pad, void* stream) {
  FVIT_CHECK(src && dst && rows > 0 && cols > 0 && cols_pad >= cols && ldd >= cols_pad,
             "fvit_cast_pad_f16: bad arguments");
  const long long total = (long long)rows * cols_pad;
  const bool vec = cols_pad % 8 == 0 && lds % 4 == 0 && ldd % 8 == 0 && cols % 4 == 0 && total / 8 < (1LL << 31) &&
                   (reinterpret_cast<uintptr_t>(src) & 15) == 0 && (reinterpret_cast<uintptr_t>(dst) & 15) == 0;
  if (vec)
    cast_pad_vec8_kernel<<<grid_for(total / 8, 256), 256, 0, (cudaStream_t)stream>>>(src, lds, (__half*)dst, ldd, rows,
                                                                                     cols, cols_pad);
  else
    cast_pad_kernel<<<grid_for(total, 256), 256, 0, (cudaStream_t)stream>>>(src, lds, (__half*)dst, ldd, rows, cols,
                                                                            cols_pad);
  return post_launch("cast_pad_kernel");
}

int fvit_cast_headpad_f16(const float* src, int64_t lds, void* dst, int64_t ldd, int32_t rows_dst,
                          int32_t cols_dst, int32_t hd, int32_t hdp, int32_t pad_rows, int32_t pad_cols,
                          void* stream) {
  FVIT_CHECK(src && dst && rows_dst > 0 && cols_dst > 0 && hd > 0 && hdp >= hd && ldd >= cols_dst,
             "fvit_cast_headpad_f16: bad arguments");
  const long long total = (long long)rows_dst * cols_dst;
  const bool vec = cols_dst % 8 == 0 && ldd % 8 == 0 && (reinterpret_cast<uintptr_t>(dst) & 15) == 0 &&
                   total / 8 < (1LL << 31) &&
                   (pad_cols ? hdp % 8 == 0 : (lds % 4 == 0 && (reinterpret_cast<uintptr_t>(src) & 15) == 0));
  if (vec)
    cast_headpad_vec8_kernel<<<grid_for(total / 8, 256), 256, 0, (cudaStream_t)stream>>>(
        src, lds, (__half*)dst, ldd, rows_dst, cols_dst, hd, hdp, pad_rows, pad_cols);
  else
    cast_headpad_kernel<<<grid_for(total, 256), 256, 0, (cudaStream_t)stream>>>(
        src, lds, (__half*)dst, ldd, rows_dst, cols_dst, hd, hdp, pad_rows, pad_cols);
  return post_launch("cast_headpad_kernel");
}

int fvit_vec_headpad_f32(const float* src, float* dst, int32_t n_dst, int32_t hd, int32_t hdp, void* stream) {
  FVIT_CHECK(src && dst && n_dst > 0 && hd > 0 && hdp >= hd, "fvit_vec_headpad_f32: bad arguments");
  vec_headpad_kernel<<<ceil_div(n_dst, 128), 128, 0, (cudaStream_t)stream>>>(src, dst, n_dst, hd, hdp);
  return post_launch("vec_headpad_kernel");
}

int fvit_pack_conv3x3_f16(const float* w, void* dst, int32_t cout, int32_t cin, int32_t kc_pad,
                          int32_t transpose_io, void* stream) {
  FVIT_CHECK(w && dst && cout > 0 && cin > 0, "fvit_pack_conv3x3_f16: bad arguments");
  FVIT_CHECK(kc_pad >= (transpose_io ? cout : cin), "fvit_pack_conv3x3_f16: kc_pad too small");
  const long long total = (long long)(transpose_io ? cin : cout) * 9 * kc_pad;
  pack_conv3x3_kernel<<<grid_for(total, 256), 256, 0, (cudaStream_t)stream>>>(
      w, (__half*)dst, cout, cin, kc_pad, transpose_io);
  return post_launch("pack_conv3x3_kernel");
}

int fvit_pack_conv3x3_taps_f16(const float* w, void* dst, int32_t cout, int32_t cin, int32_t kc_pad,
                               int32_t transpose_io, int32_t ntaps, int32_t t0, int32_t t1, int32_t t2, int32_t t3,
                               int32_t t4, int32_t t5, int32_t t6, int32_t t7, int32_t t8, void* stream) {
  FVIT_CHECK(w && dst && cout > 0 && cin > 0 && ntaps >= 1 && ntaps <= 9, "fvit_pack_conv3x3_taps_f16: bad arguments");
  FVIT_CHECK(kc_pad >= (transpose_io ? cout : cin), "fvit_pack_conv3x3_taps_f16: kc_pad too small");
  TapList tl = {{t0, t1, t2, t3, t4, t5, t6, t7, t8}};
  for (int i = 0; i < ntaps; ++i) FVIT_CHECK(tl.t[i] >= 0 && tl.t[i] < 9, "fvit_pack_conv3x3_taps_f16: bad tap");
  const long long total = (long long)(transpose_io ? cin : cout) * ntaps * kc_pad;
  pack_conv3x3_taps_kernel<<<grid_for(total, 256), 256, 0, (cudaStream_t)stream>>>(w, (__half*)dst, cout, cin, kc_pad,
                                                                                 transpose_io, ntaps, tl);
  return post_launch("pack_conv3x3_taps_kernel");
}

int fvit_affine_fold(float* scale, float* shift, int32_t n, const float* bn_w, const float* bn_b,
                     const float* bn_mean, const float* bn_var, float eps, const float* bias,
                     const float* layer_scale, void* stream) {
  FVIT_CHECK(scale && shift && n > 0, "fvit_affine_fold: bad arguments");
  FVIT_CHECK(!bn_w || (bn_b && bn_mean && bn_var), "fvit_affine_fold: incomplete BN arguments");
  affine_fold_kernel<<<ceil_div(n, 128), 128, 0, (cudaStream_t)stream>>>(
      scale, shift, n, bn_w, bn_b, bn_mean, bn_var, eps, bias, layer_scale);
  return post_launch("affine_fold_kernel");
}

int fvit_stem_conv_fwd(const float* x, int64_t sb, int64_t sc, int64_t sh, int64_t sw, int32_t B,
                       int32_t cin, int32_t H, int32_t W, const float* wgt, int32_t cout,
                       const float* scale, const float* shift, int32_t relu, const int32_t* out_row_map,
                       void* out, int64_t ldo, float* col_sum, float* col_sumsq, void* stream) {
  FVIT_CHECK(x && wgt && B > 0 && H > 0 && W > 0, "fvit_stem_conv_fwd: bad arguments");
  FVIT_CHECK(cin == 3, "fvit_stem_conv_fwd: only in_chans == 3 is supported (got %d)", cin);
  FVIT_CHECK(cout % 16 == 0 && cout <= 512, "fvit_stem_conv_fwd: cout=%d must be a multiple of 16", cout);
  FVIT_CHECK(!out || ldo % 8 == 0, "fvit_stem_conv_fwd: ldo must be a multiple of 8");
  FVIT_CHECK((col_sum == nullptr) == (col_sumsq == nullptr), "fvit_stem_conv_fwd: statistics come in pairs");
  const int Ho = (H + 1) / 2, Wo = (W + 1) / 2;
  const long long total = (long long)B * Ho * Wo * (cout / 16);
  const int block = 256;
  const long long grid = (total + block - 1) / block;
  const size_t smem = (size_t)cout * (27 + 2) * sizeof(float);
  if (smem > 48 * 1024)
    FVIT_CUDA(cudaFuncSetAttribute(stem_conv_kernel<3>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                   (int)smem));
  stem_conv_kernel<3><<<(unsigned)grid, block, smem, (cudaStream_t)stream>>>(
      x, sb, sc, sh, sw, B, H, W, wgt, cout, scale, shift, relu, out_row_map, (__half*)out, ldo,
      col_sum, col_sumsq);
  return post_launch("stem_conv_kernel");
}

int fvit_stem_im2col(const float* x, int64_t sb, int64_t sc, int64_t sh, int64_t sw, int32_t B, int32_t cin,
                     int32_t H, int32_t W, void* out, int32_t ldo, void* stream) {
  FVIT_CHECK(x && out && B > 0 && H > 0 && W > 0, "fvit_stem_im2col: bad arguments");
  FVIT_CHECK(cin >= 1 && cin <= FVIT_STEM_MAX_CIN, "fvit_stem_im2col: in_chans=%d must be in [1, %d]", cin,
             FVIT_STEM_MAX_CIN);
  const int stem_ld = (9 * cin + 31) / 32 * 32;
  FVIT_CHECK(ldo % 8 == 0 && ldo >= stem_ld, "fvit_stem_im2col: ldo=%d must be a multiple of 8 and >= %d", ldo,
             stem_ld);
  FVIT_CHECK((reinterpret_cast<uintptr_t>(out) & 15) == 0, "fvit_stem_im2col: out must be 16-byte aligned");
  const long long total = (long long)B * ((H + 1) / 2) * ((W + 1) / 2);
  FVIT_CHECK(total < (1ll << 31), "fvit_stem_im2col: too many pixels");
  if (cin != 3) {
    stem_im2col_any_kernel<<<grid_for(total * (ldo / 8), 256), 256, 0, (cudaStream_t)stream>>>(
        x, sb, sc, sh, sw, B, cin, H, W, (__half*)out, ldo);
    return post_launch("stem_im2col_any_kernel");
  }
  stem_im2col_kernel<3><<<(unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream>>>(
      x, sb, sc, sh, sw, B, H, W, (__half*)out, ldo);
  return post_launch("stem_im2col_kernel");
}

int fvit_ln_fwd(const float* x, int64_t ldx, const int32_t* in_map, int32_t rows, int32_t C,
                const float* add, int32_t group, int32_t skip, float* wb, int64_t ldwb,
                const float* gamma, const float* beta, float eps, void* out, int64_t ldo,
                const int32_t* out_map, float* mean_out, float* rstd_out, void* xhat_out, int64_t ldxh,
                void* stream) {
  FVIT_CHECK(x && gamma && beta && out && rows > 0, "fvit_ln_fwd: bad arguments");
  FVIT_CHECK(!xhat_out || ldxh % 4 == 0, "fvit_ln_fwd: xhat stride must be a multiple of 4");
  static_assert(FVIT_LN_MAX_C == 32 * 4 * 20, "the widest ln_fwd_kernel instantiation holds FVIT_LN_MAX_C channels");
  FVIT_CHECK(C % 4 == 0 && C <= FVIT_LN_MAX_C, "fvit_ln_fwd: C=%d unsupported (C %% 4 == 0, C <= %d)", C,
             FVIT_LN_MAX_C);
  FVIT_CHECK(ldx % 4 == 0 && ldo % 4 == 0 && (!wb || ldwb % 4 == 0), "fvit_ln_fwd: unaligned strides");
  FVIT_CHECK(!add || group > 0, "fvit_ln_fwd: add needs group > 0");
  const int nvec = C / 4;
  const int block = 256, wpb = block / 32;
  const int grp = group > 0 ? group : 1;
#define FVIT_LN_LAUNCH(LPR, MAXV)                                                                   \
  do {                                                                                              \
    const long long warps = ((long long)rows + (32 / LPR) - 1) / (32 / LPR);                        \
    const long long grid = (warps + wpb - 1) / wpb;                                                 \
    ln_fwd_kernel<LPR, MAXV><<<(unsigned)grid, block, 0, (cudaStream_t)stream>>>(                   \
        x, ldx, in_map, rows, C, add, grp, skip, wb, ldwb, gamma, beta, eps, (__half*)out, ldo,     \
        out_map, mean_out, rstd_out, (__half*)xhat_out, ldxh);                                      \
  } while (0)
  if (nvec <= 16) FVIT_LN_LAUNCH(8, 2);
  else if (nvec <= 32) FVIT_LN_LAUNCH(8, 4);
  else if (nvec <= 64) FVIT_LN_LAUNCH(16, 4);
  else if (nvec <= 128) FVIT_LN_LAUNCH(32, 4);
  else if (nvec <= 256) FVIT_LN_LAUNCH(32, 8);
  else if (nvec <= 512) FVIT_LN_LAUNCH(32, 16);
  else FVIT_LN_LAUNCH(32, 20);  // FasterViT-5 / -6 level 3 (2560 channels)
#undef FVIT_LN_LAUNCH
  return post_launch("ln_fwd_kernel");
}

int fvit_attn_core_fwd(const void* qkv, int64_t ldq, int32_t groups, int32_t S, int32_t heads,
                       int32_t head_dim, const float* bias, float scale, void* out, int64_t ldo,
                       float* probs_out, void* stream) {
  FVIT_CHECK(qkv && out && groups > 0 && S > 0 && heads > 0 && head_dim > 0,
             "fvit_attn_core_fwd: bad arguments");
  const int C = heads * head_dim;
  const size_t smem = ((size_t)3 * S * (head_dim + 1) + (size_t)S * (S + 1)) * sizeof(float);
  if (smem > 227 * 1024) {  // large windows (21k models): stream the keys, 64 x 64 score tiles
    FVIT_CHECK(probs_out == nullptr, "fvit_attn_core_fwd: probs_out is not available for S=%d (streaming kernel)", S);
    const size_t sm2 = ((size_t)(2 * ATT_QT + 2 * ATT_KT) * (head_dim + 1) + (size_t)ATT_QT * (ATT_KT + 1) +
                        3 * ATT_QT) * sizeof(float);
    FVIT_CHECK(sm2 <= 227 * 1024, "fvit_attn_core_fwd: head_dim=%d needs %zu B of shared memory", head_dim, sm2);
    FVIT_CHECK((long long)groups * heads <= 65535, "fvit_attn_core_fwd: groups*heads=%lld exceeds the grid limit",
               (long long)groups * heads);
    static bool stream_configured = false;
    if (!stream_configured) {
      FVIT_CUDA(cudaFuncSetAttribute(attn_stream_simt_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                     227 * 1024));
      stream_configured = true;
    }
    attn_stream_simt_kernel<<<dim3((unsigned)((S + ATT_QT - 1) / ATT_QT), (unsigned)(groups * heads)), 256, sm2,
                              (cudaStream_t)stream>>>((const __half*)qkv, ldq, S, head_dim, heads, C, bias, scale,
                                                      (__half*)out, ldo);
    return post_launch("attn_stream_simt_kernel");
  }
  static size_t configured = 0;
  if (smem > 48 * 1024 && smem > configured) {
    FVIT_CUDA(cudaFuncSetAttribute(attn_core_simt_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                   227 * 1024));
    configured = 227 * 1024;
  }
  const int block = S * S >= 4096 ? 256 : 128;
  attn_core_simt_kernel<<<(unsigned)((long long)groups * heads), block, smem, (cudaStream_t)stream>>>(
      (const __half*)qkv, ldq, S, head_dim, heads, C, bias, scale, (__half*)out, ldo, probs_out);
  return post_launch("attn_core_simt_kernel");
}

int fvit_cpb_mlp_fwd(const float* coords, int32_t P, const float* w0, const float* b0, const float* w1,
                     int32_t D, float* out, float* hidden_out, void* stream) {
  FVIT_CHECK(coords && w0 && b0 && w1 && out && P > 0 && D > 0, "fvit_cpb_mlp_fwd: bad arguments");
  if (D >= 64) {  // token embeddings: few points, many channels -> parallelise over channels
    cpb_mlp_wide_kernel<<<(D + 7) / 8, 256, 0, (cudaStream_t)stream>>>(coords, P, w0, b0, w1, D, out, hidden_out);
    return post_launch("cpb_mlp_wide_kernel");
  }
  cpb_mlp_kernel<<<P, 256, 0, (cudaStream_t)stream>>>(coords, P, w0, b0, w1, D, out, hidden_out);
  return post_launch("cpb_mlp_kernel");
}

int fvit_attn_bias_fwd(const float* table, const int64_t* index, int32_t heads, int32_t S, int32_t L,
                       float* bias, void* stream) {
  FVIT_CHECK(table && index && bias && heads > 0 && S > 0 && L > 0, "fvit_attn_bias_fwd: bad arguments");
  const long long total = (long long)heads * S * S;
  attn_bias_kernel<<<grid_for(total, 256), 256, 0, (cudaStream_t)stream>>>(
      table, (const long long*)index, heads, S, L, bias);
  return post_launch("attn_bias_kernel");
}

int fvit_token_init_fwd(const float* xs, int64_t ldx, const int32_t* pix_map, int32_t B, int32_t Hp,
                        int32_t Wp, int32_t C, const float* w, const float* bias, int32_t kh, int32_t kw,
                        int32_t sh, int32_t sw, int32_t oh, int32_t ow, const int32_t* ct_row_map,
                        float* out, int64_t ldo, void* stream) {
  FVIT_CHECK(xs && pix_map && w && bias && ct_row_map && out, "fvit_token_init_fwd: null argument");
  FVIT_CHECK((oh - 1) * sh + kh <= Hp && (ow - 1) * sw + kw <= Wp, "fvit_token_init_fwd: pool window out of range");
  const long long total = (long long)B * oh * ow * C;
  token_init_kernel<false><<<grid_for(total, 256), 256, 0, (cudaStream_t)stream>>>(
      xs, ldx, pix_map, B, Hp, Wp, C, w, bias, kh, kw, sh, sw, oh, ow, ct_row_map, out, ldo);
  return post_launch("token_init_kernel");
}

int fvit_token_init_nchw_fwd(const float* xs, int64_t ldx, const int32_t* pix_map, int32_t B, int32_t Hp,
                             int32_t Wp, int32_t C, const float* w, const float* bias, int32_t kh, int32_t kw,
                             int32_t sh, int32_t sw, int32_t oh, int32_t ow, const int32_t* ct_row_map,
                             float* out, int64_t ldo, void* stream) {
  FVIT_CHECK(xs && pix_map && w && bias && ct_row_map && out && B > 0 && C > 0 && oh > 0 && ow > 0,
             "fvit_token_init_nchw_fwd: bad arguments");
  FVIT_CHECK((oh - 1) * sh + kh <= Hp && (ow - 1) * sw + kw <= Wp, "fvit_token_init_nchw_fwd: pool window out of range");
  const long long total = (long long)B * oh * ow * C;
  token_init_kernel<true><<<grid_for(total, 256), 256, 0, (cudaStream_t)stream>>>(
      xs, ldx, pix_map, B, Hp, Wp, C, w, bias, kh, kw, sh, sw, oh, ow, ct_row_map, out, ldo);
  return post_launch("token_init_nchw_kernel");
}

int fvit_propagate_fwd(float* xs, int64_t ldx, const int32_t* src_map, int32_t rows, int32_t C,
                       const float* gamma, void* stream) {
  FVIT_CHECK(xs && src_map && rows > 0 && C % 4 == 0 && ldx % 4 == 0, "fvit_propagate_fwd: bad arguments");
  const long long total = (long long)rows * (C / 4);
  propagate_kernel<<<grid_for(total, 256), 256, 0, (cudaStream_t)stream>>>(xs, ldx, src_map, rows, C,
                                                                           gamma);
  return post_launch("propagate_kernel");
}

int fvit_pool_affine_fwd(const float* xs, int64_t ldx, const int32_t* row_map, int32_t B, int32_t T,
                         int32_t C, const float* scale, const float* shift, void* out, int64_t ldo,
                         void* stream) {
  FVIT_CHECK(xs && scale && shift && out && B > 0 && T > 0 && C % 4 == 0 && ldx % 4 == 0 && ldo % 4 == 0,
             "fvit_pool_affine_fwd: bad arguments");
  const long long total = (long long)B * (C / 4);
  pool_affine_kernel<<<grid_for(total, 128), 128, 0, (cudaStream_t)stream>>>(
      xs, ldx, row_map, B, T, C, scale, shift, (__half*)out, ldo);
  return post_launch("pool_affine_kernel");
}

int fvit_feature_map_fwd(const float* xs, int64_t ldx, const int32_t* row_map, int32_t B, int32_t T, int32_t C,
                         const float* scale, const float* shift, float* out_nchw, void* stream) {
  FVIT_CHECK(xs && scale && shift && out_nchw && B > 0 && T > 0 && C > 0 && B <= 65535,
             "fvit_feature_map_fwd: bad arguments");
  dim3 grid((T + 31) / 32, (C + 31) / 32, B);
  feature_map_kernel<<<grid, dim3(32, 8), 0, (cudaStream_t)stream>>>(xs, ldx, row_map, T, C, scale, shift, out_nchw);
  return post_launch("feature_map_kernel");
}

int fvit_nchw_pool_f16(const float* x, int32_t B, int32_t C, int32_t T, void* out16, int64_t ldo, void* stream) {
  FVIT_CHECK(x && out16 && B > 0 && C > 0 && T > 0 && ldo >= C, "fvit_nchw_pool_f16: bad arguments");
  const long long warps = (long long)B * C;
  nchw_pool_kernel<<<(unsigned)((warps * 32 + 255) / 256), 256, 0, (cudaStream_t)stream>>>(x, (int)warps, T, C,
                                                                                           (__half*)out16, ldo);
  return post_launch("nchw_pool_kernel");
}

}  // extern "C"
