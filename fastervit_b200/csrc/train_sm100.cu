// Training-path kernels (HBM-bound): batch-statistics BatchNorm (forward finalize / apply, backward),
// per-column reductions (bias / affine / layer-scale gradients), LayerNorm backward, gradient casts.
// Gradients of activations travel as fp16 tensors multiplied by a power-of-two scale that lives in
// device memory (grad_scale[0] = S, grad_scale[1] = 1/S); parameter gradients are accumulated in fp32
// and un-scaled on the fly. Contracts are in include/fvit.h.
#include <cuda_fp16.h>

#include "../../include/fvit.h"
#include "common.h"

namespace fvit {

__device__ __forceinline__ float warp_sum_t(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// ---------------------------------------------------------------------------------- column statistics
// sum[c] += sum_r d, sumsq[c] += sum_r d^2 with d = x[rows[r]][c] - K[c] over a row list (fp32 input). K = 0, or
// with `pivot` the column's first listed value (written to pivot[c]): one-pass fp32 moments about K lose
// ~ 2^-24 * (mean - K)^2 / var of the variance per term, so a pivot inside the data keeps them exact whatever
// per-channel offset the residual stream carries.
// Block = 256 threads handles a slab of rows for 64 columns: threadIdx.x & 63 = column, >> 6 = row lane.
__global__ void colstats_f32_kernel(const float* __restrict__ x, long long ldx, const int* __restrict__ rows,
                                    int nrows, int C, float* __restrict__ sum, float* __restrict__ sumsq,
                                    float* __restrict__ pivot) {
  __shared__ float red[2][4][64];
  const int c = blockIdx.y * 64 + (threadIdx.x & 63);
  const int rl = threadIdx.x >> 6;
  float s = 0.f, q = 0.f;
  if (c < C) {
    const float k = pivot ? x[(rows ? (long long)rows[0] : 0LL) * ldx + c] : 0.f;
    if (pivot && blockIdx.x == 0 && rl == 0) pivot[c] = k;
    for (int r = blockIdx.x * 4 + rl; r < nrows; r += gridDim.x * 4) {
      const long long row = rows ? rows[r] : r;
      const float v = x[row * ldx + c] - k;
      s += v;
      q += v * v;
    }
  }
  red[0][rl][threadIdx.x & 63] = s;
  red[1][rl][threadIdx.x & 63] = q;
  __syncthreads();
  if (rl == 0 && c < C) {
    const int k = threadIdx.x & 63;
    atomicAdd(sum + c, red[0][0][k] + red[0][1][k] + red[0][2][k] + red[0][3][k]);
    atomicAdd(sumsq + c, red[1][0][k] + red[1][1][k] + red[1][2][k] + red[1][3][k]);
  }
}

// BatchNorm2d training-mode finalize (fv.py:459-462, 490-493, 925 with module.training), from moments of
// d = x - K (K = pivot[c], or 0):
//   md = sum/n, var = sumsq/n - md^2 (biased, used to normalise), batch mean = K + md;
//   running_mean = (1-m) running_mean + m (K + md) ; running_var = (1-m) running_var + m var n/(n-1);
//   mean = md if the normalised data is d itself (`shifted`), else K + md;
//   scale = w * rsqrt(var+eps) [* ls] ; shift = (b - mean*scale_raw) [* ls]  -> y = data*scale + shift
__global__ void bn_finalize_kernel(const float* __restrict__ sum, const float* __restrict__ sumsq,
                                   const float* __restrict__ pivot, int shifted, float count,
                                   const float* __restrict__ w, const float* __restrict__ b, float eps,
                                   float momentum, float* __restrict__ running_mean,
                                   float* __restrict__ running_var, const float* __restrict__ ls,
                                   float* __restrict__ scale, float* __restrict__ shift,
                                   float* __restrict__ mean_out, float* __restrict__ rstd_out, int C) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  const float md = sum[c] / count;
  float var = sumsq[c] / count - md * md;
  var = fmaxf(var, 0.f);
  const float rstd = rsqrtf(var + eps);
  const float batch_mean = pivot ? pivot[c] + md : md;
  const float mean = shifted ? md : batch_mean;
  if (running_mean) {
    running_mean[c] = (1.f - momentum) * running_mean[c] + momentum * batch_mean;
    const float unbiased = count > 1.f ? var * count / (count - 1.f) : var;
    running_var[c] = (1.f - momentum) * running_var[c] + momentum * unbiased;
  }
  float s = w[c] * rstd, t = b[c] - mean * s;
  if (ls) {
    s *= ls[c];
    t *= ls[c];
  }
  scale[c] = s;
  shift[c] = t;
  if (mean_out) {
    mean_out[c] = mean;
    rstd_out[c] = rstd;
  }
}

// col_shift = bias - pivot (bias NULL = 0): the epilogue vector that centres a convolution GEMM's output and its
// statistics on the BatchNorm's pivot; recomputed every step because the bias is a trained parameter.
__global__ void bn_col_shift_kernel(const float* __restrict__ bias, const float* __restrict__ pivot, int C,
                                    float* __restrict__ col_shift) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c < C) col_shift[c] = (bias ? bias[c] : 0.f) - pivot[c];
}

// y = act(x16[row]*scale + shift) * row_scale (+ resid32[row]) for the listed rows; writes fp32 and/or fp16.
// One thread per (row, 8 channels) with 32-bit index math: one 16-byte fp16 load (the row stride is padded to a
// multiple of 8, so the last chunk of C = 196 reads its 4 padding columns too), float4 scale / shift / residual
// accesses, one 16-byte fp16 store (padding columns are written as zeros). VEC4 = every fp32 row is 16-byte aligned.
template <bool VEC4>
__global__ void __launch_bounds__(256)
affine_rows_kernel(const __half* __restrict__ x, long long ldx, const int* __restrict__ rows, int nrows, int C,
                   const float* __restrict__ scale, const float* __restrict__ shift, int act,
                   const float* __restrict__ resid, long long ldr, float* __restrict__ out32, long long ldo32,
                   __half* __restrict__ out16, long long ldo16, const float* __restrict__ row_scale) {
  const unsigned c8 = (unsigned)(C + 7) >> 3;
  const unsigned total = (unsigned)nrows * c8;
  for (unsigned i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    const unsigned ri = i / c8;
    const int j = (int)(i - ri * c8) * 8;
    const long long row = rows ? rows[ri] : (long long)ri;
    const float rsc = row_scale ? __ldg(row_scale + row) : 1.f;  // stochastic-depth mask / keep of this row
    const int nv = min(8, C - j);                                // valid channels of this chunk (4 or 8 with VEC4)
    float v[8], sc[8], sh[8], rr[8];
    {
      const uint4 pk = *reinterpret_cast<const uint4*>(x + row * ldx + j);
      const __half2* h = reinterpret_cast<const __half2*>(&pk);
#pragma unroll
      for (int u = 0; u < 4; ++u) v[2 * u] = __low2float(h[u]), v[2 * u + 1] = __high2float(h[u]);
    }
    if (VEC4) {
#pragma unroll
      for (int hf = 0; hf < 2; ++hf) {
        if (4 * hf < nv) {
          const float4 a = __ldg(reinterpret_cast<const float4*>(scale + j) + hf), b = __ldg(reinterpret_cast<const float4*>(shift + j) + hf);
          sc[4 * hf] = a.x, sc[4 * hf + 1] = a.y, sc[4 * hf + 2] = a.z, sc[4 * hf + 3] = a.w;
          sh[4 * hf] = b.x, sh[4 * hf + 1] = b.y, sh[4 * hf + 2] = b.z, sh[4 * hf + 3] = b.w;
          if (resid) {
            const float4 r4 = *(reinterpret_cast<const float4*>(resid + row * ldr + j) + hf);
            rr[4 * hf] = r4.x, rr[4 * hf + 1] = r4.y, rr[4 * hf + 2] = r4.z, rr[4 * hf + 3] = r4.w;
          }
        }
      }
    } else {
#pragma unroll
      for (int u = 0; u < 8; ++u) {
        if (u < nv) {
          sc[u] = __ldg(scale + j + u), sh[u] = __ldg(shift + j + u);
          if (resid) rr[u] = resid[row * ldr + j + u];
        }
      }
    }
#pragma unroll
    for (int u = 0; u < 8; ++u) {
      float y = 0.f;
      if (u < nv) {
        y = fmaf(v[u], sc[u], sh[u]);
        if (act == FVIT_ACT_RELU) y = fmaxf(y, 0.f);
        else if (act == FVIT_ACT_GELU) y = fvit_gelu(y);
        y *= rsc;
        if (resid) y += rr[u];
      }
      v[u] = y;
    }
    if (out32) {
      float* o = out32 + row * ldo32 + j;
      if (VEC4) {
        *reinterpret_cast<float4*>(o) = make_float4(v[0], v[1], v[2], v[3]);
        if (nv > 4) *(reinterpret_cast<float4*>(o) + 1) = make_float4(v[4], v[5], v[6], v[7]);
      } else {
#pragma unroll
        for (int u = 0; u < 8; ++u)
          if (u < nv) o[u] = v[u];
      }
    }
    if (out16) {
      __half2 h[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) h[u] = __floats2half2_rn(v[2 * u], v[2 * u + 1]);
      *reinterpret_cast<uint4*>(out16 + row * ldo16 + j) = *reinterpret_cast<const uint4*>(h);   // j + 8 <= ldo16
    }
  }
}


// ---------------------------------------------------------------------------------- gradient scaling
// gs[0] = S = 2^floor(log2(target / max|x|)), gs[1] = 1/S (single block; x is the loss gradient of the
// logits). Keeps every fp16 activation gradient inside the normal range without a host round trip.
__global__ void grad_scale_init_kernel(const float* __restrict__ x, int n, float target, float* __restrict__ gs) {
  __shared__ float red[32];
  float m = 0.f;
  for (int i = threadIdx.x; i < n; i += blockDim.x) m = fmaxf(m, fabsf(x[i]));
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = m;
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int i = 1; i < (int)(blockDim.x >> 5); ++i) m = fmaxf(m, red[i]);
    float S = 1.f;
    if (m > 0.f && isfinite(m)) S = exp2f(floorf(log2f(target / m)));
    S = fminf(fmaxf(S, 1.f / 16777216.f), 16777216.f * 65536.f);
    gs[0] = S;
    gs[1] = 1.f / S;
  }
}

// out[i] = a[i] * b[i]  (tiny vectors of device scalars, e.g. per-branch alpha = inv_scale / branch_scale)
__global__ void vec_mul_kernel(const float* a, int a_stride, const float* b, int b_stride, float* out, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = a[i * a_stride] * b[i * b_stride];
}

// out[0] = 2^-floor(log2(max|v|)) (power-of-two normaliser of a layer-scale vector), out[1] = 1/out[0]
__global__ void pow2_norm_kernel(const float* __restrict__ v, int n, float* __restrict__ out) {
  __shared__ float red[32];
  float m = 0.f;
  for (int i = threadIdx.x; i < n; i += blockDim.x) m = fmaxf(m, fabsf(v[i]));
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = m;
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int i = 1; i < (int)(blockDim.x >> 5); ++i) m = fmaxf(m, red[i]);
    float s = 1.f;
    if (m > 0.f && isfinite(m)) s = exp2f(-floorf(log2f(m)));
    out[0] = s;
    out[1] = 1.f / s;
  }
}

// out16[r][c] = (half)(x[src(r)][c] * colmul[c] * *scalar)   (fp32 -> fp16 operand cast of a gradient)
__global__ void cast_scale_f16_kernel(const float* __restrict__ x, long long ldx, const int* __restrict__ rows,
                                      int nrows, int C, const float* __restrict__ colmul,
                                      const float* __restrict__ scalar, __half* __restrict__ out, long long ldo,
                                      const float* __restrict__ row_scale) {
  const int c4 = C >> 2;
  const float sc = scalar ? __ldg(scalar) : 1.f;
  const long long total = (long long)nrows * c4;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int j = (int)(i % c4);
    const long long r = i / c4;
    const long long src = rows ? rows[r] : r;
    float4 v = reinterpret_cast<const float4*>(x + src * ldx)[j];
    const float rsc = row_scale ? sc * row_scale[r] : sc;
    float4 m = make_float4(rsc, rsc, rsc, rsc);
    if (colmul) {
      const float4 g = __ldg(reinterpret_cast<const float4*>(colmul) + j);
      m.x *= g.x, m.y *= g.y, m.z *= g.z, m.w *= g.w;
    }
    const __half2 h0 = __floats2half2_rn(v.x * m.x, v.y * m.y), h1 = __floats2half2_rn(v.z * m.z, v.w * m.w);
    uint2 pk;
    pk.x = *reinterpret_cast<const uint32_t*>(&h0);
    pk.y = *reinterpret_cast<const uint32_t*>(&h1);
    *reinterpret_cast<uint2*>(out + r * ldo + 4 * j) = pk;
  }
}

// ---------------------------------------------------------------------------------- column reductions
// out[c] += *scalar * colmul[c] * sum_r a[ra(r)][c] * (b ? b[r][c] : 1) * (row_scale ? row_scale[r] : 1)
// a is fp32 (A16 == 0) or fp16; b is fp16. Block = 32 column groups of 8 x 8 row lanes: every thread
// streams 8 consecutive columns (16-byte fp16 / 2 x 16-byte fp32 loads) over its rows, 2 rows in flight.
template <int A16>
__global__ void __launch_bounds__(256)
    colsum_kernel(const void* __restrict__ a, long long lda, const int* __restrict__ a_rows,
                  const __half* __restrict__ b, long long ldb, int nrows, int C, const float* __restrict__ colmul,
                  const float* __restrict__ scalar, float* __restrict__ out, const float* __restrict__ row_scale) {
  __shared__ float red[8][32][9];
  const int cg = threadIdx.x & 31, rl = threadIdx.x >> 5;
  const int c0 = (blockIdx.y * 32 + cg) * 8;
  float acc[8];
#pragma unroll
  for (int u = 0; u < 8; ++u) acc[u] = 0.f;
  const bool full = c0 + 8 <= C;
  if (c0 < C) {
    for (int r = blockIdx.x * 8 + rl; r < nrows; r += gridDim.x * 8) {
      const long long ra = a_rows ? a_rows[r] : r;
      float v[8];
      if (full) {
        if (A16) {
          const uint4 pk = *reinterpret_cast<const uint4*>(reinterpret_cast<const __half*>(a) + ra * lda + c0);
          const __half2* h = reinterpret_cast<const __half2*>(&pk);
#pragma unroll
          for (int u = 0; u < 4; ++u) v[2 * u] = __low2float(h[u]), v[2 * u + 1] = __high2float(h[u]);
        } else {
          const float4 p0 = *reinterpret_cast<const float4*>(reinterpret_cast<const float*>(a) + ra * lda + c0);
          const float4 p1 = *reinterpret_cast<const float4*>(reinterpret_cast<const float*>(a) + ra * lda + c0 + 4);
          v[0] = p0.x, v[1] = p0.y, v[2] = p0.z, v[3] = p0.w, v[4] = p1.x, v[5] = p1.y, v[6] = p1.z, v[7] = p1.w;
        }
        if (b) {
          const uint4 pk = *reinterpret_cast<const uint4*>(b + (long long)r * ldb + c0);
          const __half2* h = reinterpret_cast<const __half2*>(&pk);
#pragma unroll
          for (int u = 0; u < 4; ++u) v[2 * u] *= __low2float(h[u]), v[2 * u + 1] *= __high2float(h[u]);
        }
      } else {
#pragma unroll
        for (int u = 0; u < 8; ++u) {
          float x = 0.f;
          if (c0 + u < C) {
            x = A16 ? __half2float(reinterpret_cast<const __half*>(a)[ra * lda + c0 + u])
                    : reinterpret_cast<const float*>(a)[ra * lda + c0 + u];
            if (b) x *= __half2float(b[(long long)r * ldb + c0 + u]);
          }
          v[u] = x;
        }
      }
      const float rs = row_scale ? row_scale[r] : 1.f;
#pragma unroll
      for (int u = 0; u < 8; ++u) acc[u] = fmaf(v[u], rs, acc[u]);
    }
  }
#pragma unroll
  for (int u = 0; u < 8; ++u) red[rl][cg][u] = acc[u];
  __syncthreads();
  if (rl == 0 && c0 < C) {
    const float sc = scalar ? __ldg(scalar) : 1.f;
#pragma unroll
    for (int u = 0; u < 8; ++u) {
      if (c0 + u < C) {
        float s = 0.f;
#pragma unroll
        for (int k = 0; k < 8; ++k) s += red[k][cg][u];
        if (colmul) s *= colmul[c0 + u];
        atomicAdd(out + c0 + u, s * sc);
      }
    }
  }
}

// Entry of a residual-branch backward (x += gamma * f(LN(x)), fv.py:637-655) in one pass over the fp32 stream
// gradient g: dz16 = half(g * gamma * s * row_scale) (tensor-core operand of the branch's last Linear),
// dbias[c] += *bias_alpha * sum_r dz (that Linear's bias gradient) and dgamma[c] += *gamma_alpha * sum_r g * u * row_scale
// (layer-scale gradient, u = saved branch output). Replaces cast_scale_f16 + two colsum launches.
__global__ void __launch_bounds__(256)
branch_grad_kernel(const float* __restrict__ g, long long ldg, int rows, int C, const float* __restrict__ colmul,
                   const float* __restrict__ scalar, const float* __restrict__ row_scale, __half* __restrict__ dz,
                   long long lddz, const float* __restrict__ bias_alpha, float* __restrict__ dbias,
                   const __half* __restrict__ u, long long ldu, const float* __restrict__ gamma_alpha,
                   float* __restrict__ dgamma) {
  __shared__ float red[8][32][17];
  const int cg = threadIdx.x & 31, rl = threadIdx.x >> 5;
  const int c0 = (blockIdx.y * 32 + cg) * 8;
  float ab[8], ag[8];
#pragma unroll
  for (int k = 0; k < 8; ++k) ab[k] = 0.f, ag[k] = 0.f;
  if (c0 < C) {
    float cm[8];
    const float sc = scalar ? __ldg(scalar) : 1.f;
#pragma unroll
    for (int k = 0; k < 8; ++k) cm[k] = (colmul ? colmul[c0 + k] : 1.f) * sc;
#pragma unroll 2
    for (int r = blockIdx.x * 8 + rl; r < rows; r += gridDim.x * 8) {
      const float4 p0 = *reinterpret_cast<const float4*>(g + (long long)r * ldg + c0);
      const float4 p1 = *reinterpret_cast<const float4*>(g + (long long)r * ldg + c0 + 4);
      uint4 uk = make_uint4(0u, 0u, 0u, 0u);
      if (u) uk = *reinterpret_cast<const uint4*>(u + (long long)r * ldu + c0);
      const float rs = row_scale ? row_scale[r] : 1.f;
      float v[8] = {p0.x * rs, p0.y * rs, p0.z * rs, p0.w * rs, p1.x * rs, p1.y * rs, p1.z * rs, p1.w * rs};
      if (u) {
        const __half2* h = reinterpret_cast<const __half2*>(&uk);
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          ag[2 * k] = fmaf(v[2 * k], __low2float(h[k]), ag[2 * k]);
          ag[2 * k + 1] = fmaf(v[2 * k + 1], __high2float(h[k]), ag[2 * k + 1]);
        }
      }
      uint4 o;
      uint32_t* ow = reinterpret_cast<uint32_t*>(&o);
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const __half2 hv = __floats2half2_rn(v[2 * k] * cm[2 * k], v[2 * k + 1] * cm[2 * k + 1]);
        ow[k] = *reinterpret_cast<const uint32_t*>(&hv);
        ab[2 * k] += __low2float(hv), ab[2 * k + 1] += __high2float(hv);   // sum of the rounded operand values
      }
      *reinterpret_cast<uint4*>(dz + (long long)r * lddz + c0) = o;
    }
  }
#pragma unroll
  for (int k = 0; k < 8; ++k) red[rl][cg][k] = ab[k], red[rl][cg][8 + k] = ag[k];
  __syncthreads();
  // 32 column groups x 16 sums per block: one thread per (group, sum)
  for (int o = threadIdx.x; o < 32 * 16; o += 256) {
    const int grp = o >> 4, k = o & 15;
    const int c = (blockIdx.y * 32 + grp) * 8 + (k & 7);
    if (c >= C) continue;
    float s = 0.f;
#pragma unroll
    for (int q = 0; q < 8; ++q) s += red[q][grp][k];
    if (k < 8) {
      if (dbias) atomicAdd(dbias + c, s * (bias_alpha ? __ldg(bias_alpha) : 1.f));
    } else if (dgamma && u) {
      atomicAdd(dgamma + c, s * (gamma_alpha ? __ldg(gamma_alpha) : 1.f));
    }
  }
}

// out[(t - skip)][c] += *scalar * sum_w a[w*group + t][c]  for skip <= t < group (gradient of a
// positional embedding that was broadcast-added to every group; fp32 input)
__global__ void group_sum_kernel(const float* __restrict__ a, long long lda, int ngroups, int group, int skip,
                                 int C, const float* __restrict__ scalar, float* __restrict__ out) {
  const int t = blockIdx.x + skip;
  const int c = blockIdx.y * blockDim.x + threadIdx.x;
  if (c >= C) return;
  float s = 0.f;
  for (int w = blockIdx.z; w < ngroups; w += gridDim.z) s += a[((long long)w * group + t) * lda + c];
  if (scalar) s *= __ldg(scalar);
  atomicAdd(out + (long long)(t - skip) * C + c, s);
}

// ---------------------------------------------------------------------------------- LayerNorm backward
// For row r (the LayerNorm's r-th input v_r, whose forward gathered it from in_map[r] and wrote it back
// to row r):  gv = g[r] + rstd * (gam*dy - mean_c(gam*dy) - xhat * mean_c(gam*dy*xhat));
//             g[in_map[r]] = gv (and g[r] = 0 when the source is another row); dgamma += dy*xhat, dbeta += dy.
// `use_g` = 0 starts from zero instead of g[r] (first consumer of a freshly produced tensor); `clear_moved`
// zeroes g[r] when the source is another row (only meaningful when r indexes rows of g itself).
// One warp per row; per-CTA partial sums of dgamma/dbeta in shared memory, then one atomicAdd per column.
// generic (any C, scalar accesses) fallback of the vectorised kernel below
__global__ void __launch_bounds__(256)
    ln_bwd_generic_kernel(const __half* __restrict__ dy, long long lddy, const int* __restrict__ dy_map,
                  const __half* __restrict__ xhat, long long ldxh, const float* __restrict__ rstd,
                  const float* __restrict__ gamma, int rows, int C, float* __restrict__ g, long long ldg,
                  const int* __restrict__ in_map, int use_g, int clear_moved, const float* __restrict__ scalar,
                  float* __restrict__ dgamma, float* __restrict__ dbeta) {
  extern __shared__ float sh[];  // [warps][2][C]: private per-warp partial sums (lane owns column c)
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
  float* sg = sh + (size_t)warp * 2 * C;
  float* sb = sg + C;
  for (int c = lane; c < C; c += 32) {
    sg[c] = 0.f;
    sb[c] = 0.f;
  }
  for (int r = blockIdx.x * nw + warp; r < rows; r += gridDim.x * nw) {
    const long long rdy = dy_map ? dy_map[r] : r;
    if (rdy < 0) continue;  // warp-uniform
    const __half* dyr = dy + rdy * lddy;
    const __half* xr = xhat + (long long)r * ldxh;
    float s1 = 0.f, s2 = 0.f;
    for (int c = lane; c < C; c += 32) {
      const float d = __half2float(dyr[c]), xh = __half2float(xr[c]);
      const float gd = d * __ldg(gamma + c);
      s1 += gd;
      s2 += gd * xh;
      sg[c] += d * xh;
      sb[c] += d;
    }
    s1 = warp_sum_t(s1) / C;
    s2 = warp_sum_t(s2) / C;
    const float rs = rstd[r];
    const long long src = in_map ? in_map[r] : r;
    float* gr = g + (long long)r * ldg;
    float* gs_ = g + src * ldg;
    for (int c = lane; c < C; c += 32) {
      const float d = __half2float(dyr[c]), xh = __half2float(xr[c]);
      float v = rs * (d * __ldg(gamma + c) - s1 - xh * s2);
      if (use_g) v += gr[c];
      if (clear_moved && src != r) gr[c] = 0.f;
      gs_[c] = v;
    }
  }
  __syncthreads();
  const float sc = scalar ? __ldg(scalar) : 1.f;
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    float a = 0.f, b = 0.f;
    for (int w = 0; w < nw; ++w) {
      a += sh[(size_t)w * 2 * C + c];
      b += sh[(size_t)w * 2 * C + C + c];
    }
    atomicAdd(dgamma + c, a * sc);
    atomicAdd(dbeta + c, b * sc);
  }
}

// The dx half of ln_bwd_generic_kernel alone (fvit_ln_dgrad on rows the vectorised kernel does not take): no shared
// memory, no atomics.
__global__ void __launch_bounds__(256)
    ln_dgrad_generic_kernel(const __half* __restrict__ dy, long long lddy, const int* __restrict__ dy_map,
                            const __half* __restrict__ xhat, long long ldxh, const float* __restrict__ rstd,
                            const float* __restrict__ gamma, int rows, int C, float* __restrict__ g, long long ldg,
                            const int* __restrict__ in_map, int use_g, int clear_moved) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
  for (int r = blockIdx.x * nw + warp; r < rows; r += gridDim.x * nw) {
    const long long rdy = dy_map ? dy_map[r] : r;
    if (rdy < 0) continue;  // warp-uniform
    const __half* dyr = dy + rdy * lddy;
    const __half* xr = xhat + (long long)r * ldxh;
    float s1 = 0.f, s2 = 0.f;
    for (int c = lane; c < C; c += 32) {
      const float gd = __half2float(dyr[c]) * __ldg(gamma + c);
      s1 += gd;
      s2 += gd * __half2float(xr[c]);
    }
    s1 = warp_sum_t(s1) / C;
    s2 = warp_sum_t(s2) / C;
    const float rs = rstd[r];
    const long long src = in_map ? in_map[r] : r;
    float* gr = g + (long long)r * ldg;
    float* gs_ = g + src * ldg;
    for (int c = lane; c < C; c += 32) {
      float v = rs * (__half2float(dyr[c]) * __ldg(gamma + c) - s1 - __half2float(xr[c]) * s2);
      if (use_g) v += gr[c];
      if (clear_moved && src != r) gr[c] = 0.f;
      gs_[c] = v;
    }
  }
}

constexpr int LNB_MAXV = 7;       // 8-half vectors per lane: C <= 32 * 8 * 7 = 1792
constexpr int LNB_MAXV_WIDE = 10;  // FasterViT-5 / -6 level 3: C <= 32 * 8 * 10 = 2560
static_assert(32 * 8 * LNB_MAXV_WIDE == FVIT_LN_MAX_C, "the vectorised LayerNorm backward takes every fvit_ln_fwd width");
// Vectorised dx part (C % 8 == 0): one warp per row, the row's dy / xhat live in registers between the two
// passes. MAXV (vectors per lane) is a template parameter so narrow rows do not pay for wide rows' registers.
template <int MAXV, bool PREFETCH_G>
__global__ void __launch_bounds__(256)
    ln_bwd_dx_kernel(const __half* __restrict__ dy, long long lddy, const int* __restrict__ dy_map,
                     const __half* __restrict__ xhat, long long ldxh, const float* __restrict__ rstd,
                     const float* __restrict__ gamma, int rows, int C, float* __restrict__ g, long long ldg,
                     const int* __restrict__ in_map, int use_g, int clear_moved) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
  const int nv = C >> 3;
  const float invC = 1.f / (float)C;
  for (int r = blockIdx.x * nw + warp; r < rows; r += gridDim.x * nw) {
    const long long rdy = dy_map ? dy_map[r] : r;
    if (rdy < 0) continue;  // warp-uniform
    const uint4* dyr = reinterpret_cast<const uint4*>(dy + rdy * lddy);
    const uint4* xr = reinterpret_cast<const uint4*>(xhat + (long long)r * ldxh);
    float d[MAXV][8], xh[MAXV][8];
    float4 ga[MAXV][2];  // the row's incoming gradient, fetched with the operands (not after the warp reductions)
    const float4* grp = reinterpret_cast<const float4*>(g + (long long)r * ldg);
    float s1 = 0.f, s2 = 0.f;
#pragma unroll
    for (int j = 0; j < MAXV; ++j) {
      const int i = lane + 32 * j;
      if (i < nv) {
        const uint4 a = dyr[i], b = xr[i];
        if (PREFETCH_G && use_g) ga[j][0] = grp[2 * i], ga[j][1] = grp[2 * i + 1];
        const __half2* ha = reinterpret_cast<const __half2*>(&a);
        const __half2* hb = reinterpret_cast<const __half2*>(&b);
        const float4 g0 = __ldg(reinterpret_cast<const float4*>(gamma) + 2 * i);
        const float4 g1 = __ldg(reinterpret_cast<const float4*>(gamma) + 2 * i + 1);
        const float gm[8] = {g0.x, g0.y, g0.z, g0.w, g1.x, g1.y, g1.z, g1.w};
#pragma unroll
        for (int u = 0; u < 4; ++u) {
          d[j][2 * u] = __low2float(ha[u]) * gm[2 * u], d[j][2 * u + 1] = __high2float(ha[u]) * gm[2 * u + 1];
          xh[j][2 * u] = __low2float(hb[u]), xh[j][2 * u + 1] = __high2float(hb[u]);
        }
#pragma unroll
        for (int u = 0; u < 8; ++u) {
          s1 += d[j][u];
          s2 += d[j][u] * xh[j][u];
        }
      }
    }
    s1 = warp_sum_t(s1) * invC;
    s2 = warp_sum_t(s2) * invC;
    const float rs = rstd[r];
    const long long src = in_map ? in_map[r] : r;
    float* gr = g + (long long)r * ldg;
    float* gs_ = g + src * ldg;
#pragma unroll
    for (int j = 0; j < MAXV; ++j) {
      const int i = lane + 32 * j;
      if (i < nv) {
        float v[8];
#pragma unroll
        for (int u = 0; u < 8; ++u) v[u] = rs * (d[j][u] - s1 - xh[j][u] * s2);
        if (use_g) {
          const float4 a = PREFETCH_G ? ga[j][0] : grp[2 * i], b = PREFETCH_G ? ga[j][1] : grp[2 * i + 1];
          v[0] += a.x, v[1] += a.y, v[2] += a.z, v[3] += a.w, v[4] += b.x, v[5] += b.y, v[6] += b.z, v[7] += b.w;
        }
        if (clear_moved && src != r) {
          reinterpret_cast<float4*>(gr)[2 * i] = make_float4(0.f, 0.f, 0.f, 0.f);
          reinterpret_cast<float4*>(gr)[2 * i + 1] = make_float4(0.f, 0.f, 0.f, 0.f);
        }
        reinterpret_cast<float4*>(gs_)[2 * i] = make_float4(v[0], v[1], v[2], v[3]);
        reinterpret_cast<float4*>(gs_)[2 * i + 1] = make_float4(v[4], v[5], v[6], v[7]);
      }
    }
  }
}
// Parameter-gradient part: dgamma[c] += sc * sum_r dy*xhat, dbeta[c] += sc * sum_r dy. A thread owns one
// 8-column vector and walks rows; block = vpr column vectors x (256/vpr) row lanes, reduced through smem.
__global__ void __launch_bounds__(256)
    ln_bwd_param_kernel(const __half* __restrict__ dy, long long lddy, const int* __restrict__ dy_map,
                        const __half* __restrict__ xhat, long long ldxh, int rows, int C, int vpr,
                        const float* __restrict__ scalar, float* __restrict__ dgamma, float* __restrict__ dbeta) {
  __shared__ float red[256 * 17];
  const int cx = threadIdx.x % vpr, rl = threadIdx.x / vpr, RL = 256 / vpr;
  const int cv = blockIdx.y * vpr + cx;  // vector index
  float ag[8], ab[8];
#pragma unroll
  for (int u = 0; u < 8; ++u) ag[u] = 0.f, ab[u] = 0.f;
  if (cv * 8 < C) {
#pragma unroll 2
    for (int r = blockIdx.x * RL + rl; r < rows; r += gridDim.x * RL) {
      const long long rdy = dy_map ? dy_map[r] : r;
      if (rdy < 0) continue;
      const uint4 a = reinterpret_cast<const uint4*>(dy + rdy * lddy)[cv];
      const uint4 b = reinterpret_cast<const uint4*>(xhat + (long long)r * ldxh)[cv];
      const __half2* ha = reinterpret_cast<const __half2*>(&a);
      const __half2* hb = reinterpret_cast<const __half2*>(&b);
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const float2 d = __half22float2(ha[u]), x = __half22float2(hb[u]);
        ag[2 * u] += d.x * x.x, ag[2 * u + 1] += d.y * x.y;
        ab[2 * u] += d.x, ab[2 * u + 1] += d.y;
      }
    }
  }
  float* mine = red + threadIdx.x * 17;
#pragma unroll
  for (int u = 0; u < 8; ++u) mine[u] = ag[u], mine[8 + u] = ab[u];
  __syncthreads();
  // vpr*16 output sums per block; spread them over the threads
  const float sc = scalar ? __ldg(scalar) : 1.f;
  for (int o = threadIdx.x; o < vpr * 16; o += 256) {
    const int v = o >> 4, u = o & 15;
    const int c = (blockIdx.y * vpr + v) * 8 + (u & 7);
    if (c >= C) continue;
    float s = 0.f;
    for (int k = 0; k < RL; ++k) s += red[(k * vpr + v) * 17 + u];
    atomicAdd((u < 8 ? dgamma : dbeta) + c, s * sc);
  }
}

// ---------------------------------------------------------------------------------- attention backward
// One CTA per (group of S tokens, head), fp32 math, generic in S / head_dim. Recomputes P from q, k, bias;
// dV = P^T dO ; dP = dO V^T ; dS = P o (dP - rowsum(P o dP)) ; dQ = scale dS K ; dK = scale dS^T Q ;
// dbias[h] += dS. Gradients in / out are fp16 (scaled); dbias fp32 atomics (scaled).
__global__ void attn_bwd_simt_kernel(const __half* __restrict__ qkv, long long ldq, const __half* __restrict__ dout,
                                     long long lddo, int S, int hd, int hdp, int heads,
                                     const float* __restrict__ bias, float scale, __half* __restrict__ dqkv,
                                     long long lddq, float* __restrict__ dbias) {
  extern __shared__ float sm[];
  const int hp = hd + 1;
  float* sq = sm;                // [S][hd+1]
  float* sk = sq + S * hp;
  float* sv = sk + S * hp;
  float* so = sv + S * hp;       // dO
  float* sp = so + S * hp;       // [S][S+1]  P, then dS
  float* rd = sp + S * (S + 1);  // [S] rowdot
  const int g = blockIdx.x / heads, h = blockIdx.x % heads;
  const long long row0 = (long long)g * S;
  const int Cp = heads * hdp;
  for (int i = threadIdx.x; i < S * hd; i += blockDim.x) {
    const int t = i / hd, d = i % hd;
    const __half* base = qkv + (row0 + t) * ldq + h * hdp + d;
    sq[t * hp + d] = __half2float(base[0]);
    sk[t * hp + d] = __half2float(base[Cp]);
    sv[t * hp + d] = __half2float(base[2 * Cp]);
    so[t * hp + d] = __half2float(dout[(row0 + t) * lddo + h * hdp + d]);
  }
  __syncthreads();
  const float* bh = bias ? bias + (long long)h * S * S : nullptr;
  for (int i = threadIdx.x; i < S * S; i += blockDim.x) {
    const int r = i / S, c = i % S;
    float a = 0.f;
    for (int d = 0; d < hd; ++d) a = fmaf(sq[r * hp + d], sk[c * hp + d], a);
    sp[r * (S + 1) + c] = a * scale + (bh ? bh[i] : 0.f);
  }
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nwarps = blockDim.x >> 5;
  for (int r = warp; r < S; r += nwarps) {  // softmax rows
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
    s = warp_sum_t(s);
    const float inv = 1.f / s;
    for (int c = lane; c < S; c += 32) pr[c] *= inv;
  }
  __syncthreads();
  // dV[c][d] = sum_r P[r][c] dO[r][d]  -> write out immediately
  for (int i = threadIdx.x; i < S * hd; i += blockDim.x) {
    const int c = i / hd, d = i % hd;
    float a = 0.f;
    for (int r = 0; r < S; ++r) a = fmaf(sp[r * (S + 1) + c], so[r * hp + d], a);
    dqkv[(row0 + c) * lddq + 2 * Cp + h * hdp + d] = __float2half_rn(a);
  }
  // rowdot[r] = sum_c P[r][c] * (dO[r] . V[c])
  for (int r = warp; r < S; r += nwarps) {
    float acc = 0.f;
    for (int c = lane; c < S; c += 32) {
      float dp = 0.f;
      for (int d = 0; d < hd; ++d) dp = fmaf(so[r * hp + d], sv[c * hp + d], dp);
      acc = fmaf(sp[r * (S + 1) + c], dp, acc);
    }
    acc = warp_sum_t(acc);
    if (lane == 0) rd[r] = acc;
  }
  __syncthreads();
  // dS overwrites P
  for (int i = threadIdx.x; i < S * S; i += blockDim.x) {
    const int r = i / S, c = i % S;
    float dp = 0.f;
    for (int d = 0; d < hd; ++d) dp = fmaf(so[r * hp + d], sv[c * hp + d], dp);
    const float ds = sp[r * (S + 1) + c] * (dp - rd[r]);
    sp[r * (S + 1) + c] = ds;
    if (dbias) atomicAdd(dbias + (long long)h * S * S + i, ds);
  }
  __syncthreads();
  for (int i = threadIdx.x; i < S * hd; i += blockDim.x) {
    const int t = i / hd, d = i % hd;
    float aq = 0.f, ak = 0.f;
    for (int c = 0; c < S; ++c) {
      aq = fmaf(sp[t * (S + 1) + c], sk[c * hp + d], aq);   // dQ[t] = sum_c dS[t][c] K[c]
      ak = fmaf(sp[c * (S + 1) + t], sq[c * hp + d], ak);   // dK[t] = sum_r dS[r][t] Q[r]
    }
    dqkv[(row0 + t) * lddq + h * hdp + d] = __float2half_rn(aq * scale);
    dqkv[(row0 + t) * lddq + Cp + h * hdp + d] = __float2half_rn(ak * scale);
  }
  // zero the head-padding columns so padded weight-gradient GEMMs see exact zeros
  for (int i = threadIdx.x; i < S * (hdp - hd); i += blockDim.x) {
    const int t = i / (hdp - hd), d = hd + i % (hdp - hd);
#pragma unroll
    for (int w3 = 0; w3 < 3; ++w3) dqkv[(row0 + t) * lddq + w3 * Cp + h * hdp + d] = __float2half_rn(0.f);
  }
}

// ---------------------------------------------------------------------------------- small helpers
// dst[r][(c/hdp)*hd + c%hdp] (+)= *scalar * src[r][c] for c%hdp < hd (pad_cols) or rows likewise (pad_rows):
// un-pads head-padded gradient matrices into the parameter-gradient layout.
__global__ void unpad_heads_kernel(const float* __restrict__ src, long long lds, float* __restrict__ dst,
                                   long long ldd, int rows_src, int cols_src, int hd, int hdp, int pad_rows,
                                   int pad_cols, const float* __restrict__ scalar) {
  const long long total = (long long)rows_src * cols_src;
  const float sc = scalar ? __ldg(scalar) : 1.f;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int r = (int)(i / cols_src), c = (int)(i % cols_src);
    int dr = r, dc = c;
    if (pad_rows) {
      if (r % hdp >= hd) continue;
      dr = (r / hdp) * hd + r % hdp;
    }
    if (pad_cols) {
      if (c % hdp >= hd) continue;
      dc = (c / hdp) * hd + c % hdp;
    }
    dst[(long long)dr * ldd + dc] += src[(long long)r * lds + c] * sc;
  }
}

// d table[idx][h] += *scalar * dbias[h][r][c] * b (1 - b/16) with b = bias[h][r][c] = 16 sigmoid(table[idx][h])
// for r, c >= ng (backward of fvit_attn_bias_fwd; fv.py:276-299); a negative ng (S < L) skips the cropped entries
__global__ void attn_bias_bwd_kernel(const float* __restrict__ dbias, const float* __restrict__ bias,
                                     const long long* __restrict__ index, int heads, int S, int L,
                                     const float* __restrict__ scalar, float* __restrict__ dtable) {
  const int ng = S - L;
  const long long total = (long long)heads * L * L;
  const float sc = scalar ? __ldg(scalar) : 1.f;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % L), r = (int)((i / L) % L), h = (int)(i / ((long long)L * L));
    if (r + ng < 0 || c + ng < 0) continue;   // S < L: the forward cropped this part of the table away
    const long long off = ((long long)h * S + r + ng) * S + c + ng;
    const float b = bias[off];
    const float dz = dbias[off] * b * (1.f - b * (1.f / 16.f)) * sc;
    atomicAdd(dtable + index[(long long)r * L + c] * heads + h, dz);
  }
}

// Backward of fvit_cpb_mlp_fwd: dout [P, D] (fp32), hidden [P, 512] saved.
//   kernel A (grid D): dw1[d][j] += sc * sum_p dout[p][d] * hid[p][j]        (thread per j, no atomics)
//   kernel B (grid P): dhid[p][j] = (hid > 0) * sc * sum_d dout[p][d] w1[d][j]; dw0 / db0 via 3 atomics per j
__global__ void __launch_bounds__(512)
cpb_mlp_bwd_w1_kernel(int P, const float* __restrict__ hidden, const float* __restrict__ dout, int D,
                      const float* __restrict__ scalar, float* __restrict__ dw1) {
  extern __shared__ float sdo[];  // dout[:, d] (P values)
  const int d = blockIdx.x;
  const float sc = scalar ? __ldg(scalar) : 1.f;
  for (int p = threadIdx.x; p < P; p += blockDim.x) sdo[p] = dout[(long long)p * D + d] * sc;
  __syncthreads();
  const int j = threadIdx.x;  // 512 hidden units
  float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
  int p = 0;
  for (; p + 4 <= P; p += 4) {
    const float h0 = hidden[(long long)p * 512 + j], h1 = hidden[(long long)(p + 1) * 512 + j],
                h2 = hidden[(long long)(p + 2) * 512 + j], h3 = hidden[(long long)(p + 3) * 512 + j];
    a0 = fmaf(sdo[p], h0, a0), a1 = fmaf(sdo[p + 1], h1, a1), a2 = fmaf(sdo[p + 2], h2, a2),
    a3 = fmaf(sdo[p + 3], h3, a3);
  }
  for (; p < P; ++p) a0 = fmaf(sdo[p], hidden[(long long)p * 512 + j], a0);
  dw1[(long long)d * 512 + j] += (a0 + a1) + (a2 + a3);
}
// dhid[p][j] = relu'(hidden) * sum_d dout[p][d] w1[d][j] -> dw0 / db0. grid (P, 4 j-chunks, D splits): the D
// range is split because one thread's chain of dependent L2 loads is what bounds this tiny GEMV; partial
// sums are linear in the ReLU mask, so every split accumulates its share with atomics.
__global__ void __launch_bounds__(128)
cpb_mlp_bwd_kernel(const float* __restrict__ coords, int P, const float* __restrict__ w1,
                   const float* __restrict__ hidden, const float* __restrict__ dout, int D,
                   const float* __restrict__ scalar, float* __restrict__ dw0, float* __restrict__ db0) {
  extern __shared__ float sd[];  // this split's slice of the dout row
  const int p = blockIdx.x;
  const int j = blockIdx.y * 128 + threadIdx.x;
  const int d0 = (int)((long long)D * blockIdx.z / gridDim.z), d1 = (int)((long long)D * (blockIdx.z + 1) / gridDim.z);
  const float sc = scalar ? __ldg(scalar) : 1.f;
  for (int d = d0 + threadIdx.x; d < d1; d += blockDim.x) sd[d - d0] = dout[(long long)p * D + d] * sc;
  __syncthreads();
  const float hv = hidden[(long long)p * 512 + j];
  if (hv <= 0.f) return;
  const float* wp = w1 + (long long)d0 * 512 + j;
  const int n = d1 - d0;
  float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
  int d = 0;
  for (; d + 8 <= n; d += 8) {
    const float v0 = wp[(long long)d * 512], v1 = wp[(long long)(d + 1) * 512], v2 = wp[(long long)(d + 2) * 512],
                v3 = wp[(long long)(d + 3) * 512], v4 = wp[(long long)(d + 4) * 512], v5 = wp[(long long)(d + 5) * 512],
                v6 = wp[(long long)(d + 6) * 512], v7 = wp[(long long)(d + 7) * 512];
    a0 = fmaf(sd[d], v0, a0), a1 = fmaf(sd[d + 1], v1, a1), a2 = fmaf(sd[d + 2], v2, a2), a3 = fmaf(sd[d + 3], v3, a3);
    a0 = fmaf(sd[d + 4], v4, a0), a1 = fmaf(sd[d + 5], v5, a1), a2 = fmaf(sd[d + 6], v6, a2), a3 = fmaf(sd[d + 7], v7, a3);
  }
  for (; d < n; ++d) a0 = fmaf(sd[d], wp[(long long)d * 512], a0);
  const float dh = (a0 + a1) + (a2 + a3);
  atomicAdd(dw0 + 2 * j, dh * coords[2 * p]);
  atomicAdd(dw0 + 2 * j + 1, dh * coords[2 * p + 1]);
  atomicAdd(db0 + j, dh);
}

// Backward of the head: y[b,t,c] = xhat*w + beta with batch statistics, pooled[b,c] = mean_t y.
// reduce: s1[c] = sum_b dp[b,c] ; s2[c] = sum_b dp[b,c]/T * sum_t xhat[b,t,c]   (dp = d pooled, scaled)
__global__ void pool_bn_bwd_reduce_kernel(const float* __restrict__ xs, long long ldx, const int* __restrict__ rows,
                                          int B, int T, int C, const float* __restrict__ mean,
                                          const float* __restrict__ rstd, const float* __restrict__ dpool,
                                          long long lddp, float* __restrict__ s1, float* __restrict__ s2) {
  const int c = blockIdx.y * blockDim.x + threadIdx.x;
  if (c >= C) return;
  float a1 = 0.f, a2 = 0.f;
  for (int b = blockIdx.x; b < B; b += gridDim.x) {
    const float d = dpool[(long long)b * lddp + c];
    float sx = 0.f;
    for (int t = 0; t < T; ++t) {
      const long long row = rows ? rows[(long long)b * T + t] : (long long)b * T + t;
      sx += (xs[row * ldx + c] - mean[c]) * rstd[c];
    }
    a1 += d;
    a2 += d / T * sx;
  }
  atomicAdd(s1 + c, a1);
  atomicAdd(s2 + c, a2);
}
// apply: g[row(b,t)][c] = w*rstd*(dp[b,c]/T - s1/N - xhat*s2/N) ; dw = s2 * inv, dbeta = s1 * inv (block 0)
__global__ void pool_bn_bwd_apply_kernel(const float* __restrict__ xs, long long ldx, const int* __restrict__ rows,
                                         int B, int T, int C, const float* __restrict__ mean,
                                         const float* __restrict__ rstd, const float* __restrict__ w,
                                         const float* __restrict__ dpool, long long lddp,
                                         const float* __restrict__ s1, const float* __restrict__ s2,
                                         const float* __restrict__ scalar, float* __restrict__ g, long long ldg,
                                         float* __restrict__ dw, float* __restrict__ dbeta) {
  const long long total = (long long)B * T * C;
  const float N = (float)B * T;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % C);
    const long long bt = i / C;
    const int b = (int)(bt / T);
    const long long row = rows ? rows[bt] : bt;
    const float xh = (xs[row * ldx + c] - mean[c]) * rstd[c];
    g[row * ldg + c] = w[c] * rstd[c] * (dpool[(long long)b * lddp + c] / T - s1[c] / N - xh * s2[c] / N);
  }
  if (blockIdx.x == 0) {
    const float sc = scalar ? __ldg(scalar) : 1.f;
    for (int c = threadIdx.x; c < C; c += blockDim.x) {
      dw[c] += s2[c] * sc;
      dbeta[c] += s1[c] * sc;
    }
  }
}

// dst[map[r]][c] += src[r][c]  (fp32; map entries < 0 skipped). Carrier-token gradient back to the window
// layout (ct_dewindow backward).
__global__ void scatter_add_rows_kernel(const float* __restrict__ src, long long lds, float* __restrict__ dst,
                                        long long ldd, const int* __restrict__ map, int rows, int C) {
  const int c4 = C >> 2;
  const long long total = (long long)rows * c4;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int j = (int)(i % c4);
    const long long r = i / c4;
    const int d = map[r];
    if (d < 0) continue;
    const float4 v = reinterpret_cast<const float4*>(src + r * lds)[j];
    float4* o = reinterpret_cast<float4*>(dst + (long long)d * ldd) + j;
    float4 t = *o;
    t.x += v.x, t.y += v.y, t.z += v.z, t.w += v.w;
    *o = t;
  }
}

// ---------------------------------------------------------------------------------- BatchNorm backward
// y = act(xhat*w + b) with xhat = (raw - mean)*rstd over the listed rows; dyv = upstream gradient
// (fp32 g rows or fp16 rows) times colmul (layer scale), masked by the activation derivative
// (ReLU: y > 0; GELU handled by the caller's GEMM epilogue, act = NONE here).
// reduce: s1[c] += sum dy ; s2[c] += sum dy * xhat
template <int G16>
__global__ void bn_bwd_reduce_kernel(const void* __restrict__ gin, long long ldg, const int* __restrict__ g_rows,
                                     const __half* __restrict__ raw, long long ldr, const int* __restrict__ r_rows,
                                     int nrows, int C, const float* __restrict__ mean, const float* __restrict__ rstd,
                                     const float* __restrict__ w, const float* __restrict__ b, int act,
                                     const float* __restrict__ colmul, float* __restrict__ s1, float* __restrict__ s2,
                                     const float* __restrict__ row_scale) {
  __shared__ float red[2][4][64];
  const int c = blockIdx.y * 64 + (threadIdx.x & 63);
  const int rl = threadIdx.x >> 6;
  float a1 = 0.f, a2 = 0.f;
  if (c < C) {
    const float mu = mean[c], rs = rstd[c], wc = w[c], bc = b[c], cm = colmul ? colmul[c] : 1.f;
    for (int r = blockIdx.x * 4 + rl; r < nrows; r += gridDim.x * 4) {
      const long long rg = g_rows ? g_rows[r] : r, rr = r_rows ? r_rows[r] : r;
      float dy = G16 ? __half2float(reinterpret_cast<const __half*>(gin)[rg * ldg + c])
                     : reinterpret_cast<const float*>(gin)[rg * ldg + c];
      const float xh = (__half2float(raw[rr * ldr + c]) - mu) * rs;
      dy *= cm;
      if (row_scale) dy *= row_scale[rg];
      if (act == FVIT_ACT_RELU && fmaf(xh, wc, bc) <= 0.f) dy = 0.f;
      a1 += dy;
      a2 += dy * xh;
    }
  }
  red[0][rl][threadIdx.x & 63] = a1;
  red[1][rl][threadIdx.x & 63] = a2;
  __syncthreads();
  if (rl == 0 && c < C) {
    const int k = threadIdx.x & 63;
    atomicAdd(s1 + c, red[0][0][k] + red[0][1][k] + red[0][2][k] + red[0][3][k]);
    atomicAdd(s2 + c, red[1][0][k] + red[1][1][k] + red[1][2][k] + red[1][3][k]);
  }
}
// apply: dx16[orow][c] = w*rstd*(dy - s1/N - xhat*s2/N); block 0 also emits dw += s2*sc, db += s1*sc
template <int G16>
__global__ void bn_bwd_apply_kernel(const void* __restrict__ gin, long long ldg, const int* __restrict__ g_rows,
                                    const __half* __restrict__ raw, long long ldr, const int* __restrict__ r_rows,
                                    int nrows, int C, float count, const float* __restrict__ mean,
                                    const float* __restrict__ rstd, const float* __restrict__ w,
                                    const float* __restrict__ b, int act, const float* __restrict__ colmul,
                                    const float* __restrict__ s1, const float* __restrict__ s2,
                                    const float* __restrict__ scalar, __half* __restrict__ out, long long ldo,
                                    const int* __restrict__ o_rows, float* __restrict__ dw, float* __restrict__ db,
                                    const float* __restrict__ row_scale) {
  const long long total = (long long)nrows * C;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % C);
    const long long r = i / C;
    const long long rg = g_rows ? g_rows[r] : r, rr = r_rows ? r_rows[r] : r, ro = o_rows ? o_rows[r] : r;
    float dy = G16 ? __half2float(reinterpret_cast<const __half*>(gin)[rg * ldg + c])
                   : reinterpret_cast<const float*>(gin)[rg * ldg + c];
    const float xh = (__half2float(raw[rr * ldr + c]) - mean[c]) * rstd[c];
    if (colmul) dy *= colmul[c];
    if (row_scale) dy *= row_scale[rg];
    if (act == FVIT_ACT_RELU && fmaf(xh, w[c], b[c]) <= 0.f) dy = 0.f;
    out[ro * ldo + c] = __float2half_rn(w[c] * rstd[c] * (dy - s1[c] / count - xh * s2[c] / count));
  }
  if (blockIdx.x == 0) {
    const float sc = scalar ? __ldg(scalar) : 1.f;
    for (int c = threadIdx.x; c < C; c += blockDim.x) {
      dw[c] += s2[c] * sc;
      db[c] += s1[c] * sc;
    }
  }
}

// Vectorised variants (C % 4 == 0, all leading dimensions % 4 == 0): each thread owns 4 adjacent channels, keeps
// their constants in registers and walks rows with 8/16-byte accesses. Block = vpr column vectors x (256/vpr) rows.
template <int G16>
__device__ __forceinline__ float4 bn_load_dy4(const void* gin, long long off) {
  if (G16) {
    const uint2 u = *reinterpret_cast<const uint2*>(reinterpret_cast<const __half*>(gin) + off);
    const float2 a = __half22float2(*reinterpret_cast<const __half2*>(&u.x));
    const float2 b = __half22float2(*reinterpret_cast<const __half2*>(&u.y));
    return make_float4(a.x, a.y, b.x, b.y);
  }
  return *reinterpret_cast<const float4*>(reinterpret_cast<const float*>(gin) + off);
}
__device__ __forceinline__ float4 bn_load_h4(const __half* p) {
  const uint2 u = *reinterpret_cast<const uint2*>(p);
  const float2 a = __half22float2(*reinterpret_cast<const __half2*>(&u.x));
  const float2 b = __half22float2(*reinterpret_cast<const __half2*>(&u.y));
  return make_float4(a.x, a.y, b.x, b.y);
}
template <int G16>
__global__ void __launch_bounds__(256, 3)
bn_bwd_reduce_v4_kernel(const void* __restrict__ gin, long long ldg, const int* __restrict__ g_rows,
                        const __half* __restrict__ raw, long long ldr, const int* __restrict__ r_rows, int nrows, int C,
                        int vpr, const float* __restrict__ mean, const float* __restrict__ rstd,
                        const float* __restrict__ w, const float* __restrict__ b, int act,
                        const float* __restrict__ colmul, float* __restrict__ s1, float* __restrict__ s2,
                        const float* __restrict__ row_scale) {
  __shared__ float4 red[2][256];
  const int cx = threadIdx.x % vpr, rl = threadIdx.x / vpr, RL = 256 / vpr;
  const int c = (blockIdx.y * vpr + cx) * 4;
  float4 a1 = make_float4(0.f, 0.f, 0.f, 0.f), a2 = a1;
  if (c < C) {
    const float4 mu = *reinterpret_cast<const float4*>(mean + c), rs = *reinterpret_cast<const float4*>(rstd + c);
    const float4 wc = *reinterpret_cast<const float4*>(w + c), bc = *reinterpret_cast<const float4*>(b + c);
    const float4 cm = colmul ? *reinterpret_cast<const float4*>(colmul + c) : make_float4(1.f, 1.f, 1.f, 1.f);
    const bool relu = act == FVIT_ACT_RELU;
    const bool same_rows = g_rows == r_rows;
    const int rstep = gridDim.x * RL;
    // 4 rows per trip: all index loads, then all data loads, then the math (memory-level parallelism)
    for (int r0 = blockIdx.x * RL + rl; r0 < nrows; r0 += 4 * rstep) {
      long long rg[4], rr[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const int r = r0 + u * rstep;
        rg[u] = r < nrows ? (g_rows ? (long long)g_rows[r] : (long long)r) : -1;
        rr[u] = same_rows ? rg[u] : (r < nrows ? (r_rows ? (long long)r_rows[r] : (long long)r) : -1);
      }
      float4 dy[4], x[4];
      float rsc[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        if (rg[u] >= 0) {
          dy[u] = bn_load_dy4<G16>(gin, rg[u] * ldg + c);
          x[u] = bn_load_h4(raw + rr[u] * ldr + c);
          rsc[u] = row_scale ? row_scale[rg[u]] : 1.f;
        } else {
          dy[u] = make_float4(0.f, 0.f, 0.f, 0.f);
          x[u] = make_float4(0.f, 0.f, 0.f, 0.f);
          rsc[u] = 0.f;
        }
      }
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const float xh0 = (x[u].x - mu.x) * rs.x, xh1 = (x[u].y - mu.y) * rs.y, xh2 = (x[u].z - mu.z) * rs.z,
                    xh3 = (x[u].w - mu.w) * rs.w;
        float4 d = dy[u];
        d.x *= cm.x * rsc[u], d.y *= cm.y * rsc[u], d.z *= cm.z * rsc[u], d.w *= cm.w * rsc[u];
        if (relu) {
          if (fmaf(xh0, wc.x, bc.x) <= 0.f) d.x = 0.f;
          if (fmaf(xh1, wc.y, bc.y) <= 0.f) d.y = 0.f;
          if (fmaf(xh2, wc.z, bc.z) <= 0.f) d.z = 0.f;
          if (fmaf(xh3, wc.w, bc.w) <= 0.f) d.w = 0.f;
        }
        a1.x += d.x, a1.y += d.y, a1.z += d.z, a1.w += d.w;
        a2.x += d.x * xh0, a2.y += d.y * xh1, a2.z += d.z * xh2, a2.w += d.w * xh3;
      }
    }
  }
  red[0][threadIdx.x] = a1;
  red[1][threadIdx.x] = a2;
  __syncthreads();
  if (rl == 0 && c < C) {
    for (int k = 1; k < RL; ++k) {
      const float4 u = red[0][k * vpr + cx], v = red[1][k * vpr + cx];
      a1.x += u.x, a1.y += u.y, a1.z += u.z, a1.w += u.w;
      a2.x += v.x, a2.y += v.y, a2.z += v.z, a2.w += v.w;
    }
    atomicAdd(s1 + c, a1.x), atomicAdd(s1 + c + 1, a1.y), atomicAdd(s1 + c + 2, a1.z), atomicAdd(s1 + c + 3, a1.w);
    atomicAdd(s2 + c, a2.x), atomicAdd(s2 + c + 1, a2.y), atomicAdd(s2 + c + 2, a2.z), atomicAdd(s2 + c + 3, a2.w);
  }
}
template <int G16>
__global__ void __launch_bounds__(256, 3)
bn_bwd_apply_v4_kernel(const void* __restrict__ gin, long long ldg, const int* __restrict__ g_rows,
                       const __half* __restrict__ raw, long long ldr, const int* __restrict__ r_rows, int nrows, int C,
                       int vpr, float inv_count, const float* __restrict__ mean, const float* __restrict__ rstd,
                       const float* __restrict__ w, const float* __restrict__ b, int act,
                       const float* __restrict__ colmul, const float* __restrict__ s1, const float* __restrict__ s2,
                       const float* __restrict__ scalar, __half* __restrict__ out, long long ldo,
                       const int* __restrict__ o_rows, float* __restrict__ dw, float* __restrict__ db,
                       const float* __restrict__ row_scale) {
  const int cx = threadIdx.x % vpr, rl = threadIdx.x / vpr, RL = 256 / vpr;
  const int c = (blockIdx.y * vpr + cx) * 4;
  if (c >= C) return;
  const float4 mu = *reinterpret_cast<const float4*>(mean + c), rs = *reinterpret_cast<const float4*>(rstd + c);
  const float4 wc = *reinterpret_cast<const float4*>(w + c), bc = *reinterpret_cast<const float4*>(b + c);
  const float4 cm = colmul ? *reinterpret_cast<const float4*>(colmul + c) : make_float4(1.f, 1.f, 1.f, 1.f);
  const float4 t1 = *reinterpret_cast<const float4*>(s1 + c), t2 = *reinterpret_cast<const float4*>(s2 + c);
  const float m1x = t1.x * inv_count, m1y = t1.y * inv_count, m1z = t1.z * inv_count, m1w = t1.w * inv_count;
  const float m2x = t2.x * inv_count, m2y = t2.y * inv_count, m2z = t2.z * inv_count, m2w = t2.w * inv_count;
  const float kx = wc.x * rs.x, ky = wc.y * rs.y, kz = wc.z * rs.z, kw = wc.w * rs.w;
  const bool relu = act == FVIT_ACT_RELU;
  const bool same_rows = g_rows == r_rows, same_out = o_rows == g_rows;
  const int rstep = gridDim.x * RL;
  for (int r0 = blockIdx.x * RL + rl; r0 < nrows; r0 += 4 * rstep) {
    long long rg[4], rr[4], ro[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const int r = r0 + u * rstep;
      const bool ok = r < nrows;
      rg[u] = ok ? (g_rows ? (long long)g_rows[r] : (long long)r) : -1;
      rr[u] = same_rows ? rg[u] : (ok ? (r_rows ? (long long)r_rows[r] : (long long)r) : -1);
      ro[u] = same_out ? rg[u] : (ok ? (o_rows ? (long long)o_rows[r] : (long long)r) : -1);
    }
    float4 dy[4], x[4];
    float rsc[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      if (rg[u] >= 0) {
        dy[u] = bn_load_dy4<G16>(gin, rg[u] * ldg + c);
        x[u] = bn_load_h4(raw + rr[u] * ldr + c);
        rsc[u] = row_scale ? row_scale[rg[u]] : 1.f;
      } else {
        dy[u] = make_float4(0.f, 0.f, 0.f, 0.f);
        x[u] = make_float4(0.f, 0.f, 0.f, 0.f);
        rsc[u] = 0.f;
      }
    }
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      if (rg[u] < 0) continue;
      const float xh0 = (x[u].x - mu.x) * rs.x, xh1 = (x[u].y - mu.y) * rs.y, xh2 = (x[u].z - mu.z) * rs.z,
                  xh3 = (x[u].w - mu.w) * rs.w;
      float4 d = dy[u];
      d.x *= cm.x * rsc[u], d.y *= cm.y * rsc[u], d.z *= cm.z * rsc[u], d.w *= cm.w * rsc[u];
      if (relu) {
        if (fmaf(xh0, wc.x, bc.x) <= 0.f) d.x = 0.f;
        if (fmaf(xh1, wc.y, bc.y) <= 0.f) d.y = 0.f;
        if (fmaf(xh2, wc.z, bc.z) <= 0.f) d.z = 0.f;
        if (fmaf(xh3, wc.w, bc.w) <= 0.f) d.w = 0.f;
      }
      const __half2 o0 = __floats2half2_rn(kx * (d.x - m1x - xh0 * m2x), ky * (d.y - m1y - xh1 * m2y));
      const __half2 o1 = __floats2half2_rn(kz * (d.z - m1z - xh2 * m2z), kw * (d.w - m1w - xh3 * m2w));
      uint2 o;
      o.x = *reinterpret_cast<const uint32_t*>(&o0);
      o.y = *reinterpret_cast<const uint32_t*>(&o1);
      *reinterpret_cast<uint2*>(out + ro[u] * ldo + c) = o;
    }
  }
  if (blockIdx.x == 0 && rl == 0) {
    const float sc = scalar ? __ldg(scalar) : 1.f;
    dw[c] += t2.x * sc, dw[c + 1] += t2.y * sc, dw[c + 2] += t2.z * sc, dw[c + 3] += t2.w * sc;
    db[c] += t1.x * sc, db[c + 1] += t1.y * sc, db[c + 2] += t1.z * sc, db[c + 3] += t1.w * sc;
  }
}

// ---- 8-channel (16-byte fp16 / 2 x float4 fp32) versions: a lane owns 8 channels of a row, vpr lanes cover a row
// (C = 196 -> 25 chunks -> 32 lanes), 256 / vpr rows per block pass, two rows per trip. Rows are padded to multiples
// of 8 columns, so the last chunk reads (and writes, as zeros) its padding columns.
// a row's 8-channel chunk is held packed (uint4 of halves, or two float4) between the load and the math so that four
// rows can be in flight per thread without spilling
template <int G16>
struct BnDy8 {
  uint4 a, b;  // G16: a = 8 halves; fp32: a, b = 2 x 4 floats
  __device__ __forceinline__ void load(const void* g, long long off, int nv) {
    if (G16) {
      a = *reinterpret_cast<const uint4*>(reinterpret_cast<const __half*>(g) + off);
    } else {
      const uint4* p4 = reinterpret_cast<const uint4*>(reinterpret_cast<const float*>(g) + off);
      a = p4[0];
      b = nv > 4 ? p4[1] : make_uint4(0u, 0u, 0u, 0u);
    }
  }
  __device__ __forceinline__ void zero() { a = b = make_uint4(0u, 0u, 0u, 0u); }
  __device__ __forceinline__ void unpack(float (&d)[8]) const {
    if (G16) {
      const __half2* h = reinterpret_cast<const __half2*>(&a);
#pragma unroll
      for (int u = 0; u < 4; ++u) d[2 * u] = __low2float(h[u]), d[2 * u + 1] = __high2float(h[u]);
    } else {
      d[0] = __uint_as_float(a.x), d[1] = __uint_as_float(a.y), d[2] = __uint_as_float(a.z), d[3] = __uint_as_float(a.w);
      d[4] = __uint_as_float(b.x), d[5] = __uint_as_float(b.y), d[6] = __uint_as_float(b.z), d[7] = __uint_as_float(b.w);
    }
  }
};
__device__ __forceinline__ void bn_unpack_x8(const uint4& pk, float (&x)[8]) {
  const __half2* h = reinterpret_cast<const __half2*>(&pk);
#pragma unroll
  for (int u = 0; u < 4; ++u) x[2 * u] = __low2float(h[u]), x[2 * u + 1] = __high2float(h[u]);
}
struct BnCols8 {
  float mu[8], rs[8], wc[8], bc[8], cm[8];
};
__device__ __forceinline__ void bn_load_cols8(BnCols8& k, int c, int nv, const float* mean, const float* rstd, const float* w,
                                              const float* b, const float* colmul) {
#pragma unroll
  for (int u = 0; u < 8; ++u) {
    const bool in = u < nv;
    k.mu[u] = in ? __ldg(mean + c + u) : 0.f, k.rs[u] = in ? __ldg(rstd + c + u) : 0.f;
    k.wc[u] = in ? __ldg(w + c + u) : 0.f, k.bc[u] = in ? __ldg(b + c + u) : 0.f;
    k.cm[u] = in ? (colmul ? __ldg(colmul + c + u) : 1.f) : 0.f;
  }
}
constexpr int BN8_ROWS = 4;  // rows per trip: all index loads, then all data loads, then the math
template <int G16>
__global__ void __launch_bounds__(256, 2)
bn_bwd_reduce_v8_kernel(const void* __restrict__ gin, long long ldg, const int* __restrict__ g_rows,
                        const __half* __restrict__ raw, long long ldr, const int* __restrict__ r_rows, int nrows, int C,
                        int vpr, const float* __restrict__ mean, const float* __restrict__ rstd,
                        const float* __restrict__ w, const float* __restrict__ b, int act,
                        const float* __restrict__ colmul, float* __restrict__ s1, float* __restrict__ s2,
                        const float* __restrict__ row_scale) {
  __shared__ float red[2][8][257];
  const int cx = threadIdx.x % vpr, rl = threadIdx.x / vpr, RL = 256 / vpr;
  const int c = (blockIdx.y * vpr + cx) * 8;
  const int nv = min(8, C - c);
  float a1[8], a2[8];
#pragma unroll
  for (int u = 0; u < 8; ++u) a1[u] = a2[u] = 0.f;
  if (nv > 0) {
    BnCols8 k;
    bn_load_cols8(k, c, nv, mean, rstd, w, b, colmul);
    const bool relu = act == FVIT_ACT_RELU;
    const bool same_rows = g_rows == r_rows;
    const int rstep = gridDim.x * RL;
    for (int r0 = blockIdx.x * RL + rl; r0 < nrows; r0 += BN8_ROWS * rstep) {
      long long rg[BN8_ROWS], rr[BN8_ROWS];
#pragma unroll
      for (int t = 0; t < BN8_ROWS; ++t) {
        const int r = r0 + t * rstep;
        rg[t] = r < nrows ? (g_rows ? (long long)g_rows[r] : (long long)r) : -1;
        rr[t] = same_rows ? rg[t] : (r < nrows ? (r_rows ? (long long)r_rows[r] : (long long)r) : -1);
      }
      BnDy8<G16> dyp[BN8_ROWS];
      uint4 xp[BN8_ROWS];
      float rsc[BN8_ROWS];
#pragma unroll
      for (int t = 0; t < BN8_ROWS; ++t) {
        if (rg[t] >= 0) {
          dyp[t].load(gin, rg[t] * ldg + c, nv);
          xp[t] = *reinterpret_cast<const uint4*>(raw + rr[t] * ldr + c);
          rsc[t] = row_scale ? row_scale[rg[t]] : 1.f;
        } else {
          dyp[t].zero();
          xp[t] = make_uint4(0u, 0u, 0u, 0u);
          rsc[t] = 0.f;
        }
      }
#pragma unroll
      for (int t = 0; t < BN8_ROWS; ++t) {
        float dyt[8], xt[8];
        dyp[t].unpack(dyt);
        bn_unpack_x8(xp[t], xt);
#pragma unroll
        for (int u = 0; u < 8; ++u) {
          const float xh = (xt[u] - k.mu[u]) * k.rs[u];
          float d = dyt[u] * k.cm[u] * rsc[t];
          if (relu && fmaf(xh, k.wc[u], k.bc[u]) <= 0.f) d = 0.f;
          a1[u] += d;
          a2[u] = fmaf(d, xh, a2[u]);
        }
      }
    }
  }
#pragma unroll
  for (int u = 0; u < 8; ++u) red[0][u][threadIdx.x] = a1[u], red[1][u][threadIdx.x] = a2[u];
  __syncthreads();
  // 2 x 8 x vpr column sums of RL partials each
  for (int q = threadIdx.x; q < 16 * vpr; q += 256) {
    const int which = q / (8 * vpr), u = (q / vpr) & 7, lane = q % vpr;
    const int cc = (blockIdx.y * vpr + lane) * 8 + u;
    if (cc < C) {
      float t = 0.f;
      for (int kk = 0; kk < RL; ++kk) t += red[which][u][kk * vpr + lane];
      atomicAdd((which ? s2 : s1) + cc, t);
    }
  }
}
template <int G16>
__global__ void __launch_bounds__(256, 2)
bn_bwd_apply_v8_kernel(const void* __restrict__ gin, long long ldg, const int* __restrict__ g_rows,
                       const __half* __restrict__ raw, long long ldr, const int* __restrict__ r_rows, int nrows, int C,
                       int vpr, float inv_count, const float* __restrict__ mean, const float* __restrict__ rstd,
                       const float* __restrict__ w, const float* __restrict__ b, int act,
                       const float* __restrict__ colmul, const float* __restrict__ s1, const float* __restrict__ s2,
                       const float* __restrict__ scalar, __half* __restrict__ out, long long ldo,
                       const int* __restrict__ o_rows, float* __restrict__ dw, float* __restrict__ db,
                       const float* __restrict__ row_scale) {
  const int cx = threadIdx.x % vpr, rl = threadIdx.x / vpr, RL = 256 / vpr;
  const int c = (blockIdx.y * vpr + cx) * 8;
  const int nv = min(8, C - c);
  if (nv <= 0) return;
  BnCols8 k;
  bn_load_cols8(k, c, nv, mean, rstd, w, b, colmul);
  float m1[8], m2[8], kk[8], t1[8], t2[8];
#pragma unroll
  for (int u = 0; u < 8; ++u) {
    t1[u] = u < nv ? s1[c + u] : 0.f, t2[u] = u < nv ? s2[c + u] : 0.f;
    m1[u] = t1[u] * inv_count, m2[u] = t2[u] * inv_count, kk[u] = k.wc[u] * k.rs[u];
  }
  const bool relu = act == FVIT_ACT_RELU;
  const bool same_rows = g_rows == r_rows, same_out = o_rows == g_rows;
  const int rstep = gridDim.x * RL;
  for (int r0 = blockIdx.x * RL + rl; r0 < nrows; r0 += BN8_ROWS * rstep) {
    long long rg[BN8_ROWS], rr[BN8_ROWS], ro[BN8_ROWS];
#pragma unroll
    for (int t = 0; t < BN8_ROWS; ++t) {
      const int r = r0 + t * rstep;
      const bool ok = r < nrows;
      rg[t] = ok ? (g_rows ? (long long)g_rows[r] : (long long)r) : -1;
      rr[t] = same_rows ? rg[t] : (ok ? (r_rows ? (long long)r_rows[r] : (long long)r) : -1);
      ro[t] = same_out ? rg[t] : (ok ? (o_rows ? (long long)o_rows[r] : (long long)r) : -1);
    }
    BnDy8<G16> dyp[BN8_ROWS];
    uint4 xp[BN8_ROWS];
    float rsc[BN8_ROWS];
#pragma unroll
    for (int t = 0; t < BN8_ROWS; ++t) {
      if (rg[t] >= 0) {
        dyp[t].load(gin, rg[t] * ldg + c, nv);
        xp[t] = *reinterpret_cast<const uint4*>(raw + rr[t] * ldr + c);
        rsc[t] = row_scale ? row_scale[rg[t]] : 1.f;
      }
    }
#pragma unroll
    for (int t = 0; t < BN8_ROWS; ++t) {
      if (rg[t] < 0) continue;
      float o[8], dyt[8], xt[8];
      dyp[t].unpack(dyt);
      bn_unpack_x8(xp[t], xt);
#pragma unroll
      for (int u = 0; u < 8; ++u) {
        const float xh = (xt[u] - k.mu[u]) * k.rs[u];
        float d = dyt[u] * k.cm[u] * rsc[t];
        if (relu && fmaf(xh, k.wc[u], k.bc[u]) <= 0.f) d = 0.f;
        o[u] = u < nv ? kk[u] * (d - m1[u] - xh * m2[u]) : 0.f;
      }
      __half2 h[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) h[u] = __floats2half2_rn(o[2 * u], o[2 * u + 1]);
      *reinterpret_cast<uint4*>(out + ro[t] * ldo + c) = *reinterpret_cast<const uint4*>(h);
    }
  }
  if (blockIdx.x == 0 && rl == 0) {
    const float sc = scalar ? __ldg(scalar) : 1.f;
#pragma unroll
    for (int u = 0; u < 8; ++u)
      if (u < nv) dw[c + u] += t2[u] * sc, db[c + u] += t1[u] * sc;
  }
}

// conv weight gradient repack: dst[co][ci][tap] += src[co][tap * cin + ci] (src row stride ld)
__global__ void unpack_conv_grad_kernel(const float* __restrict__ src, int ld, float* __restrict__ dst, int cout,
                                        int cin) {
  const long long total = (long long)cout * cin * 9;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int tap = (int)(i % 9);
    const int ci = (int)((i / 9) % cin);
    const int co = (int)(i / (9LL * cin));
    dst[i] += src[(long long)co * ld + tap * cin + ci];
  }
}

// Element of the carrier gradient that belongs to pooled value (b, c, o = y0*ow + x0): channel c of row
// ct_row_map[b*nout + o], or -- kNchwTokens, the detection backbone's NCHW read-back (fvit_token_init_nchw_fwd) --
// channel f % C of row ct_row_map[b*nout + f / C] with f = c*nout + o.
template <bool kNchwTokens>
__device__ __forceinline__ long long ct_grad_at(const int* __restrict__ ct_row_map, int b, int o, int nout, int c, int C,
                                                long long ldg) {
  if (kNchwTokens) {
    const long long f = (long long)c * nout + o;
    return (long long)ct_row_map[(long long)b * nout + f / C] * ldg + f % C;
  }
  return (long long)ct_row_map[(long long)b * nout + o] * ldg + c;
}

// TokenInitializer backward: for ct[b, (y0,x0), c] = bias + mean_{pool window} dwconv3x3(x):
//   dx[pixel] += sum over pooled outputs / taps ; dw[c][tap] += ... ; dbias[c] += sum gct. One thread per
//   (b, pixel, channel) gathers from the (at most few) pooled outputs that cover the pixel's 3x3 halo.
template <bool kNchwTokens>
__global__ void token_init_bwd_kernel(const float* __restrict__ g, long long ldg, const int* __restrict__ pix_map,
                                      const int* __restrict__ ct_row_map, int B, int Hp, int Wp, int C,
                                      const float* __restrict__ w, int kh, int kw, int sh, int sw, int oh, int ow,
                                      float* __restrict__ gx, long long ldgx) {
  // blockIdx.x / threadIdx.x walk channels, blockIdx.y walks pixels: 32-bit index math only
  const float inv = 1.f / (float)(kh * kw);
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  const int npos = B * Hp * Wp;
  for (int pos = blockIdx.y; pos < npos; pos += gridDim.y) {
    const int x = pos % Wp, y = (pos / Wp) % Hp, b = pos / (Wp * Hp);
    const int row = pix_map[pos];
    if (row < 0) continue;
    float acc = 0.f;
    // pixel (y,x) feeds conv output (cy,cx) = (y - r + 1, x - s + 1) with tap (r,s); that conv pixel is
    // pooled into every output (y0,x0) with y0*sh <= cy < y0*sh + kh
    for (int r = 0; r < 3; ++r)
      for (int s = 0; s < 3; ++s) {
        const int cy = y - r + 1, cx = x - s + 1;
        if (cy < 0 || cy >= Hp || cx < 0 || cx >= Wp) continue;
        const float wt = w[c * 9 + r * 3 + s] * inv;
        // pooled outputs covering conv pixel (cy, cx): y0*sh <= cy < y0*sh + kh
        const int y0lo = cy - kh + sh >= 0 ? (cy - kh + sh) / sh : 0, y0hi = min(oh - 1, cy / sh);
        const int x0lo = cx - kw + sw >= 0 ? (cx - kw + sw) / sw : 0, x0hi = min(ow - 1, cx / sw);
        for (int y0 = y0lo; y0 <= y0hi; ++y0)
          for (int x0 = x0lo; x0 <= x0hi; ++x0) {
            acc = fmaf(wt, g[ct_grad_at<kNchwTokens>(ct_row_map, b, y0 * ow + x0, oh * ow, c, C, ldg)], acc);
          }
      }
    gx[(long long)row * ldgx + c] += acc;
  }
}
// Same result for maps that fit in shared memory (every 224-class model: 14 x 14 pixels, 4 x 4 carriers): one CTA
// per (image, 32 channels) stages the carrier gradients, forms the average-pool backward d conv[pixel] once
// (instead of once per tap: 36 gathers per element in the kernel above) and applies the 9-tap transpose of the
// depthwise convolution out of shared memory. Thread = (channel lane, pixel lane): 128-byte row accesses.
template <bool kNchwTokens>
__global__ void __launch_bounds__(256)
token_init_bwd_tile_kernel(const float* __restrict__ g, long long ldg, const int* __restrict__ pix_map,
                           const int* __restrict__ ct_row_map, int Hp, int Wp, int C, const float* __restrict__ w,
                           int kh, int kw, int sh, int sw, int oh, int ow, float* __restrict__ gx, long long ldgx) {
  extern __shared__ float tsm[];
  float* sg = tsm;                 // [oh*ow][32] carrier-row gradients of this image
  float* sd = tsm + oh * ow * 32;  // [Hp*Wp][32] d loss / d conv output
  const int b = blockIdx.y, cl = threadIdx.x & 31, pl = threadIdx.x >> 5;
  const int c = blockIdx.x * 32 + cl;
  const bool cok = c < C;
  const int nout = oh * ow, npix = Hp * Wp;
  for (int o = pl; o < nout; o += 8)
    sg[o * 32 + cl] = cok ? g[ct_grad_at<kNchwTokens>(ct_row_map, b, o, nout, c, C, ldg)] : 0.f;
  __syncthreads();
  const float inv = 1.f / (float)(kh * kw);
  for (int p = pl; p < npix; p += 8) {
    const int cy = p / Wp, cx = p - cy * Wp;
    // pooled outputs covering conv pixel (cy, cx): y0*sh <= cy < y0*sh + kh
    const int y0lo = cy - kh + sh >= 0 ? (cy - kh + sh) / sh : 0, y0hi = min(oh - 1, cy / sh);
    const int x0lo = cx - kw + sw >= 0 ? (cx - kw + sw) / sw : 0, x0hi = min(ow - 1, cx / sw);
    float a = 0.f;
    for (int y0 = y0lo; y0 <= y0hi; ++y0)
      for (int x0 = x0lo; x0 <= x0hi; ++x0) a += sg[(y0 * ow + x0) * 32 + cl];
    sd[p * 32 + cl] = a * inv;
  }
  __syncthreads();
  if (!cok) return;
  float wl[9];
#pragma unroll
  for (int t = 0; t < 9; ++t) wl[t] = __ldg(w + c * 9 + t);
  for (int p = pl; p < npix; p += 8) {
    const int y = p / Wp, x = p - y * Wp;
    const int row = pix_map[b * npix + p];
    if (row < 0) continue;
    float acc = 0.f;
#pragma unroll
    for (int r = 0; r < 3; ++r) {
      const int cy = y - r + 1;
      if (cy < 0 || cy >= Hp) continue;
#pragma unroll
      for (int s2 = 0; s2 < 3; ++s2) {
        const int cx = x - s2 + 1;
        if (cx < 0 || cx >= Wp) continue;
        acc = fmaf(wl[r * 3 + s2], sd[(cy * Wp + cx) * 32 + cl], acc);
      }
    }
    gx[(long long)row * ldgx + c] += acc;
  }
}
// dw[c][tap] += sc * sum_{b,y0,x0} gct * mean_pool x[.. + tap - 1] ; dbias[c] += sc * sum gct
template <bool kNchwTokens>
__global__ void token_init_wgrad_kernel(const float* __restrict__ g, long long ldg, const __half* __restrict__ xs,
                                        long long ldx, const int* __restrict__ pix_map,
                                        const int* __restrict__ ct_row_map, int B, int Hp, int Wp, int C, int kh,
                                        int kw, int sh, int sw, int oh, int ow, const float* __restrict__ scalar,
                                        float* __restrict__ dw, float* __restrict__ dbias) {
  __shared__ float red[3][10][128];
  const int cl = threadIdx.x & 127, lane_p = threadIdx.x >> 7;  // 128 channels x 4 position lanes
  const int c = blockIdx.x * 128 + cl;
  const float inv = 1.f / (float)(kh * kw);
  float acc[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
  float ab = 0.f;
  if (c < C) {
    for (long long pos = blockIdx.y * 4 + lane_p; pos < (long long)B * oh * ow; pos += gridDim.y * 4) {
      const int x0 = (int)(pos % ow), y0 = (int)((pos / ow) % oh), b = (int)(pos / ((long long)ow * oh));
      const float gv = g[ct_grad_at<kNchwTokens>(ct_row_map, b, y0 * ow + x0, oh * ow, c, C, ldg)];
      ab += gv;
      // dw[tap] += gv/(kh kw) * sum over the pool window of x[conv pixel + tap - 1]: walk the (kh+2) x (kw+2) input
      // patch once and add each pixel to the (up to 9) taps that see it
      for (int py = -1; py <= kh; ++py) {
        const int iy = y0 * sh + py;
        if (iy < 0 || iy >= Hp) continue;
        for (int px = -1; px <= kw; ++px) {
          const int ix = x0 * sw + px;
          if (ix < 0 || ix >= Wp) continue;
          const int row = pix_map[((long long)b * Hp + iy) * Wp + ix];
          if (row < 0) continue;
          const float xv = gv * inv * __half2float(xs[(long long)row * ldx + c]);
          // input pixel offset py = conv offset (py - r + 1) must lie in [0, kh): r in [py - kh + 2, py + 1]
#pragma unroll
          for (int r = 0; r < 3; ++r)
#pragma unroll
            for (int s = 0; s < 3; ++s)
              if (py - r + 1 >= 0 && py - r + 1 < kh && px - s + 1 >= 0 && px - s + 1 < kw) acc[r * 3 + s] += xv;
        }
      }
    }
  }
  if (lane_p > 0) {
#pragma unroll
    for (int t9 = 0; t9 < 9; ++t9) red[lane_p - 1][t9][cl] = acc[t9];
    red[lane_p - 1][9][cl] = ab;
  }
  __syncthreads();
  if (lane_p == 0 && c < C) {
    const float sc = scalar ? __ldg(scalar) : 1.f;
#pragma unroll
    for (int t9 = 0; t9 < 9; ++t9)
      atomicAdd(dw + c * 9 + t9, (acc[t9] + red[0][t9][cl] + red[1][t9][cl] + red[2][t9][cl]) * sc);
    atomicAdd(dbias + c, (ab + red[0][9][cl] + red[1][9][cl] + red[2][9][cl]) * sc);
  }
}

// Backward of fvit_propagate_fwd (x[r] += gamma * x[src[r]]): g[src[r]] += gamma * g[r] (atomics: a carrier
// row collects ~ws^2/ct^2 token rows) and dgamma[c] += *scalar * sum_r g[r][c] * x[src[r]][c].
__global__ void propagate_bwd_kernel(float* __restrict__ g, long long ldg, const float* __restrict__ xs, long long ldx,
                                     const int* __restrict__ src_map, int rows, int C, const float* __restrict__ gamma,
                                     const float* __restrict__ scalar, float* __restrict__ dgamma) {
  __shared__ float red[4][64];
  const int c = blockIdx.y * 64 + (threadIdx.x & 63);
  const int rl = threadIdx.x >> 6;
  float acc = 0.f;
  if (c < C) {
    const float gm = gamma ? gamma[c] : 1.f;
    for (int r = blockIdx.x * 4 + rl; r < rows; r += gridDim.x * 4) {
      const int s = src_map[r];
      if (s < 0) continue;
      const float gv = g[(long long)r * ldg + c];
      atomicAdd(g + (long long)s * ldg + c, gm * gv);
      acc = fmaf(gv, xs[(long long)s * ldx + c], acc);
    }
  }
  red[rl][threadIdx.x & 63] = acc;
  __syncthreads();
  if (rl == 0 && c < C && dgamma) {
    const int k = threadIdx.x & 63;
    const float sc = scalar ? __ldg(scalar) : 1.f;
    atomicAdd(dgamma + c, (red[0][k] + red[1][k] + red[2][k] + red[3][k]) * sc);
  }
}

static inline int grid_cap(long long total, int block, int per_sm) {
  long long g = (total + block - 1) / block;
  const long long cap = (long long)num_sms() * per_sm;
  if (g > cap) g = cap;
  if (g < 1) g = 1;
  return (int)g;
}

}  // namespace fvit

using namespace fvit;

extern "C" {

int fvit_colstats_f32(const float* x, int64_t ldx, const int32_t* rows, int32_t nrows, int32_t C, float* sum,
                      float* sumsq, void* stream) {
  FVIT_CHECK(x && sum && sumsq && nrows > 0 && C > 0, "fvit_colstats_f32: bad arguments");
  dim3 grid((unsigned)grid_cap(((long long)nrows + 15) / 16, 1, 24), (unsigned)((C + 63) / 64));
  colstats_f32_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(x, ldx, rows, nrows, C, sum, sumsq, nullptr);
  return post_launch("colstats_f32_kernel");
}

int fvit_colstats_pivot_f32(const float* x, int64_t ldx, const int32_t* rows, int32_t nrows, int32_t C, float* pivot,
                            float* sum, float* sumsq, void* stream) {
  FVIT_CHECK(x && pivot && sum && sumsq && nrows > 0 && C > 0, "fvit_colstats_pivot_f32: bad arguments");
  dim3 grid((unsigned)grid_cap(((long long)nrows + 15) / 16, 1, 24), (unsigned)((C + 63) / 64));
  colstats_f32_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(x, ldx, rows, nrows, C, sum, sumsq, pivot);
  return post_launch("colstats_f32_kernel");
}

static int bn_finalize_launch(const float* sum, const float* sumsq, const float* pivot, int32_t shifted, float count,
                              const float* w, const float* b, float eps, float momentum, float* running_mean,
                              float* running_var, const float* layer_scale, float* scale, float* shift, float* mean_out,
                              float* rstd_out, int32_t C, void* stream) {
  FVIT_CHECK(sum && sumsq && w && b && scale && shift && C > 0 && count > 0, "fvit_bn_finalize: bad arguments");
  FVIT_CHECK((running_mean == nullptr) == (running_var == nullptr), "fvit_bn_finalize: running stats come in pairs");
  FVIT_CHECK((mean_out == nullptr) == (rstd_out == nullptr), "fvit_bn_finalize: mean/rstd outputs come in pairs");
  bn_finalize_kernel<<<ceil_div(C, 128), 128, 0, (cudaStream_t)stream>>>(
      sum, sumsq, pivot, shifted, count, w, b, eps, momentum, running_mean, running_var, layer_scale, scale, shift,
      mean_out, rstd_out, C);
  return post_launch("bn_finalize_kernel");
}

int fvit_bn_finalize(const float* sum, const float* sumsq, float count, const float* w, const float* b, float eps,
                     float momentum, float* running_mean, float* running_var, const float* layer_scale,
                     float* scale, float* shift, float* mean_out, float* rstd_out, int32_t C, void* stream) {
  return bn_finalize_launch(sum, sumsq, nullptr, 0, count, w, b, eps, momentum, running_mean, running_var, layer_scale,
                            scale, shift, mean_out, rstd_out, C, stream);
}

int fvit_bn_finalize_pivot(const float* sum, const float* sumsq, const float* pivot, int32_t shifted, float count,
                           const float* w, const float* b, float eps, float momentum, float* running_mean,
                           float* running_var, const float* layer_scale, float* scale, float* shift, float* mean_out,
                           float* rstd_out, int32_t C, void* stream) {
  FVIT_CHECK(pivot != nullptr, "fvit_bn_finalize_pivot: pivot is required");
  return bn_finalize_launch(sum, sumsq, pivot, shifted, count, w, b, eps, momentum, running_mean, running_var,
                            layer_scale, scale, shift, mean_out, rstd_out, C, stream);
}

int fvit_bn_col_shift(const float* bias, const float* pivot, int32_t C, float* col_shift, void* stream) {
  FVIT_CHECK(pivot && col_shift && C > 0, "fvit_bn_col_shift: bad arguments");
  bn_col_shift_kernel<<<ceil_div(C, 128), 128, 0, (cudaStream_t)stream>>>(bias, pivot, C, col_shift);
  return post_launch("bn_col_shift_kernel");
}

int fvit_affine_rows(const void* x16, int64_t ldx, const int32_t* rows, int32_t nrows, int32_t C,
                     const float* scale, const float* shift, int32_t act, const float* resid, int64_t ldr,
                     float* out32, int64_t ldo32, void* out16, int64_t ldo16, const float* row_scale, void* stream) {
  FVIT_CHECK(x16 && scale && shift && nrows > 0 && C > 0 && (out32 || out16), "fvit_affine_rows: bad arguments");
  FVIT_CHECK(ldx % 8 == 0 && (!out16 || ldo16 % 8 == 0), "fvit_affine_rows: fp16 strides must be multiples of 8");
  const long long total = (long long)nrows * ((C + 7) / 8);
  FVIT_CHECK(total < (1LL << 31), "fvit_affine_rows: %lld chunks exceed the 32-bit index range", total);
  FVIT_CHECK((reinterpret_cast<uintptr_t>(x16) & 15) == 0 && (!out16 || (reinterpret_cast<uintptr_t>(out16) & 15) == 0),
             "fvit_affine_rows: fp16 buffers must be 16-byte aligned");
  // float4 accesses of the fp32 vectors / rows: C % 4 == 0 keeps every 8-chunk at 4 or 8 valid channels
  const bool vec4 = C % 4 == 0 && (reinterpret_cast<uintptr_t>(scale) & 15) == 0 && (reinterpret_cast<uintptr_t>(shift) & 15) == 0 &&
                    (!resid || (ldr % 4 == 0 && (reinterpret_cast<uintptr_t>(resid) & 15) == 0)) &&
                    (!out32 || (ldo32 % 4 == 0 && (reinterpret_cast<uintptr_t>(out32) & 15) == 0));
  const int grid = grid_cap(total, 256, 16);
  if (vec4)
    affine_rows_kernel<true><<<grid, 256, 0, (cudaStream_t)stream>>>((const __half*)x16, ldx, rows, nrows, C, scale, shift, act,
                                                                     resid, ldr, out32, ldo32, (__half*)out16, ldo16, row_scale);
  else
    affine_rows_kernel<false><<<grid, 256, 0, (cudaStream_t)stream>>>((const __half*)x16, ldx, rows, nrows, C, scale, shift, act,
                                                                      resid, ldr, out32, ldo32, (__half*)out16, ldo16, row_scale);
  return post_launch("affine_rows_kernel");
}

int fvit_grad_scale_init(const float* x, int32_t n, float target, float* gs, void* stream) {
  FVIT_CHECK(x && gs && n > 0 && target > 0, "fvit_grad_scale_init: bad arguments");
  grad_scale_init_kernel<<<1, 1024, 0, (cudaStream_t)stream>>>(x, n, target, gs);
  return post_launch("grad_scale_init_kernel");
}

int fvit_vec_mul(const float* a, int32_t a_stride, const float* b, int32_t b_stride, float* out, int32_t n,
                 void* stream) {
  FVIT_CHECK(a && b && out && n > 0, "fvit_vec_mul: bad arguments");
  vec_mul_kernel<<<ceil_div(n, 128), 128, 0, (cudaStream_t)stream>>>(a, a_stride, b, b_stride, out, n);
  return post_launch("vec_mul_kernel");
}

int fvit_pow2_norm(const float* v, int32_t n, float* out, void* stream) {
  FVIT_CHECK(v && out && n > 0, "fvit_pow2_norm: bad arguments");
  pow2_norm_kernel<<<1, 256, 0, (cudaStream_t)stream>>>(v, n, out);
  return post_launch("pow2_norm_kernel");
}

int fvit_cast_scale_f16(const float* x, int64_t ldx, const int32_t* rows, int32_t nrows, int32_t C,
                        const float* colmul, const float* scalar, void* out, int64_t ldo, const float* row_scale,
                        void* stream) {
  FVIT_CHECK(x && out && nrows > 0 && C > 0 && C % 4 == 0 && ldx % 4 == 0 && ldo % 4 == 0,
             "fvit_cast_scale_f16: bad arguments");
  const long long total = (long long)nrows * (C / 4);
  cast_scale_f16_kernel<<<grid_cap(total, 256, 16), 256, 0, (cudaStream_t)stream>>>(
      x, ldx, rows, nrows, C, colmul, scalar, (__half*)out, ldo, row_scale);
  return post_launch("cast_scale_f16_kernel");
}

int fvit_colsum(const void* a, int32_t a_is_f16, int64_t lda, const int32_t* a_rows, const void* b16, int64_t ldb,
                int32_t nrows, int32_t C, const float* colmul, const float* scalar, float* out, const float* row_scale,
                void* stream) {
  FVIT_CHECK(a && out && nrows > 0 && C > 0, "fvit_colsum: bad arguments");
  FVIT_CHECK(lda % (a_is_f16 ? 8 : 4) == 0 && (!b16 || ldb % 8 == 0) && (reinterpret_cast<uintptr_t>(a) & 15) == 0,
             "fvit_colsum: rows must be 16-byte aligned");
  const unsigned gy = (unsigned)((C + 255) / 256);
  long long gx = ((long long)num_sms() * 8 + gy - 1) / gy;
  const long long gx_max = ((long long)nrows + 31) / 32;
  if (gx > gx_max) gx = gx_max;
  if (gx < 1) gx = 1;
  dim3 grid((unsigned)gx, gy);
  if (a_is_f16)
    colsum_kernel<1><<<grid, 256, 0, (cudaStream_t)stream>>>(a, lda, a_rows, (const __half*)b16, ldb, nrows, C,
                                                             colmul, scalar, out, row_scale);
  else
    colsum_kernel<0><<<grid, 256, 0, (cudaStream_t)stream>>>(a, lda, a_rows, (const __half*)b16, ldb, nrows, C,
                                                             colmul, scalar, out, row_scale);
  return post_launch("colsum_kernel");
}

int fvit_branch_grad(const float* g, int64_t ldg, int32_t rows, int32_t C, const float* colmul, const float* scalar,
                     const float* row_scale, void* dz16, int64_t lddz, const float* bias_alpha, float* dbias,
                     const void* u16, int64_t ldu, const float* gamma_alpha, float* dgamma, void* stream) {
  FVIT_CHECK(g && dz16 && rows > 0 && C > 0 && C % 8 == 0 && ldg % 4 == 0 && lddz % 8 == 0 && (!u16 || ldu % 8 == 0) &&
                 (reinterpret_cast<uintptr_t>(g) & 15) == 0 && (reinterpret_cast<uintptr_t>(dz16) & 15) == 0 &&
                 (!u16 || (reinterpret_cast<uintptr_t>(u16) & 15) == 0),
             "fvit_branch_grad: needs C %% 8 == 0 and 16-byte aligned rows");
  const unsigned gy = (unsigned)((C + 255) / 256);
  long long gx = ((long long)num_sms() * 8 + gy - 1) / gy;
  const long long gx_max = ((long long)rows + 31) / 32;
  if (gx > gx_max) gx = gx_max;
  if (gx < 1) gx = 1;
  branch_grad_kernel<<<dim3((unsigned)gx, gy), 256, 0, (cudaStream_t)stream>>>(
      g, ldg, rows, C, colmul, scalar, row_scale, (__half*)dz16, lddz, bias_alpha, dbias, (const __half*)u16, ldu,
      gamma_alpha, dgamma);
  return post_launch("branch_grad_kernel");
}

int fvit_group_sum(const float* a, int64_t lda, int32_t ngroups, int32_t group, int32_t skip, int32_t C,
                   const float* scalar, float* out, void* stream) {
  FVIT_CHECK(a && out && ngroups > 0 && group > skip && skip >= 0 && C > 0, "fvit_group_sum: bad arguments");
  int z = ngroups < 32 ? ngroups : 32;
  dim3 grid((unsigned)(group - skip), (unsigned)((C + 127) / 128), (unsigned)z);
  group_sum_kernel<<<grid, 128, 0, (cudaStream_t)stream>>>(a, lda, ngroups, group, skip, C, scalar, out);
  return post_launch("group_sum_kernel");
}

// the vectorised dx kernel of a LayerNorm backward (fvit_ln_bwd, fvit_ln_dgrad); the caller checked the layout
static void ln_dx_launch(const __half* dyh, int64_t lddy, const int32_t* dy_map, const __half* xhh, int64_t ldxh,
                         const float* rstd, const float* gamma, int32_t rows, int32_t C, float* g, int64_t ldg,
                         const int32_t* in_map, int32_t use_g, int32_t clear_moved, cudaStream_t st) {
  const int block = 256, wpb = 8;
  long long grid = ((long long)rows + wpb - 1) / wpb;
  const long long cap = (long long)num_sms() * 16;
  if (grid > cap) grid = cap;
  const int nvl = (C / 8 + 31) / 32;
  // up to LNB_MAXV vectors per lane, g is fetched with the operands instead of after the warp reductions
#define FVIT_LN_DX(MV, PF)                                                                                          \
  ln_bwd_dx_kernel<MV, PF><<<(unsigned)grid, block, 0, st>>>(dyh, lddy, dy_map, xhh, ldxh, rstd, gamma, rows, C, g, ldg, \
                                                             in_map, use_g, clear_moved)
  if (nvl <= 1) FVIT_LN_DX(1, true);
  else if (nvl <= 2) FVIT_LN_DX(2, true);
  else if (nvl <= 4) FVIT_LN_DX(4, true);
  else if (nvl <= LNB_MAXV) FVIT_LN_DX(LNB_MAXV, true);
  else FVIT_LN_DX(LNB_MAXV_WIDE, false);  // prefetching g at ten vectors per lane spills past 255 registers
#undef FVIT_LN_DX
}

int fvit_ln_bwd(const void* dy16, int64_t lddy, const int32_t* dy_map, const void* xhat16, int64_t ldxh,
                const float* rstd, const float* gamma, int32_t rows, int32_t C, float* g, int64_t ldg,
                const int32_t* in_map, int32_t use_g, int32_t clear_moved, const float* scalar, float* dgamma,
                float* dbeta, void* stream) {
  FVIT_CHECK(dy16 && xhat16 && rstd && gamma && g && dgamma && dbeta && rows > 0 && C > 0,
             "fvit_ln_bwd: bad arguments");
  const bool vec = C % 8 == 0 && C <= 32 * 8 * LNB_MAXV_WIDE && lddy % 8 == 0 && ldxh % 8 == 0 && ldg % 4 == 0;
  const int block = 256, wpb = 8;
  long long grid = ((long long)rows + wpb - 1) / wpb;
  const cudaStream_t st = (cudaStream_t)stream;
  if (vec) {
    const __half* dyh = (const __half*)dy16;
    const __half* xhh = (const __half*)xhat16;
    ln_dx_launch(dyh, lddy, dy_map, xhh, ldxh, rstd, gamma, rows, C, g, ldg, in_map, use_g, clear_moved, st);
    int vpr = 1;
    while (vpr < 32 && vpr < C / 8) vpr *= 2;
    const unsigned gy = (unsigned)((C / 8 + vpr - 1) / vpr);
    const int RL = 256 / vpr;
    long long gx = ((long long)num_sms() * 8 + gy - 1) / gy;
    const long long gx_max = ((long long)rows + RL * 4 - 1) / (RL * 4);
    if (gx > gx_max) gx = gx_max;
    if (gx < 1) gx = 1;
    ln_bwd_param_kernel<<<dim3((unsigned)gx, gy), 256, 0, st>>>(dyh, lddy, dy_map, xhh, ldxh, rows, C, vpr, scalar, dgamma,
                                                                dbeta);
    return post_launch("ln_bwd kernels");
  }
  const long long cap = (long long)num_sms() * 8;
  if (grid > cap) grid = cap;
  const size_t smem = (size_t)wpb * 2 * C * sizeof(float);
  static bool configured = false;
  if (smem > 48 * 1024 && !configured) {
    FVIT_CUDA(cudaFuncSetAttribute(ln_bwd_generic_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    configured = true;
  }
  ln_bwd_generic_kernel<<<(unsigned)grid, block, smem, st>>>((const __half*)dy16, lddy, dy_map, (const __half*)xhat16,
                                                             ldxh, rstd, gamma, rows, C, g, ldg, in_map, use_g,
                                                             clear_moved, scalar, dgamma, dbeta);
  return post_launch("ln_bwd_kernel");
}

int fvit_ln_dgrad(const void* dy16, int64_t lddy, const int32_t* dy_map, const void* xhat16, int64_t ldxh,
                  const float* rstd, const float* gamma, int32_t rows, int32_t C, float* g, int64_t ldg,
                  const int32_t* in_map, int32_t use_g, int32_t clear_moved, void* stream) {
  FVIT_CHECK(dy16 && xhat16 && rstd && gamma && g && rows > 0 && C > 0, "fvit_ln_dgrad: bad arguments");
  const cudaStream_t st = (cudaStream_t)stream;
  if (C % 8 == 0 && C <= 32 * 8 * LNB_MAXV_WIDE && lddy % 8 == 0 && ldxh % 8 == 0 && ldg % 4 == 0) {
    ln_dx_launch((const __half*)dy16, lddy, dy_map, (const __half*)xhat16, ldxh, rstd, gamma, rows, C, g, ldg, in_map,
                 use_g, clear_moved, st);
    return post_launch("ln_bwd_dx_kernel");
  }
  long long grid = ((long long)rows + 7) / 8;
  const long long cap = (long long)num_sms() * 8;
  if (grid > cap) grid = cap;
  ln_dgrad_generic_kernel<<<(unsigned)grid, 256, 0, st>>>((const __half*)dy16, lddy, dy_map, (const __half*)xhat16, ldxh,
                                                          rstd, gamma, rows, C, g, ldg, in_map, use_g, clear_moved);
  return post_launch("ln_dgrad_generic_kernel");
}

int fvit_attn_core_bwd(const void* qkv, int64_t ldq, const void* dout, int64_t lddo, int32_t groups, int32_t S,
                       int32_t heads, int32_t head_dim, int32_t hdp, const float* bias, float scale, void* dqkv,
                       int64_t lddq, float* dbias, void* stream) {
  FVIT_CHECK(qkv && dout && dqkv && groups > 0 && S > 0 && heads > 0 && head_dim > 0 && hdp >= head_dim,
             "fvit_attn_core_bwd: bad arguments");
  const size_t smem = ((size_t)4 * S * (head_dim + 1) + (size_t)S * (S + 1) + S) * sizeof(float);
  FVIT_CHECK(smem <= 227 * 1024, "fvit_attn_core_bwd: S=%d head_dim=%d needs %zu B of shared memory", S, head_dim,
             smem);
  static bool configured = false;
  if (smem > 48 * 1024 && !configured) {
    FVIT_CUDA(cudaFuncSetAttribute(attn_bwd_simt_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
    configured = true;
  }
  attn_bwd_simt_kernel<<<(unsigned)((long long)groups * heads), 256, smem, (cudaStream_t)stream>>>(
      (const __half*)qkv, ldq, (const __half*)dout, lddo, S, head_dim, hdp, heads, bias, scale, (__half*)dqkv, lddq,
      dbias);
  return post_launch("attn_bwd_simt_kernel");
}

int fvit_unpad_heads_f32(const float* src, int64_t lds, float* dst, int64_t ldd, int32_t rows_src, int32_t cols_src,
                         int32_t hd, int32_t hdp, int32_t pad_rows, int32_t pad_cols, const float* scalar,
                         void* stream) {
  FVIT_CHECK(src && dst && rows_src > 0 && cols_src > 0 && hd > 0 && hdp >= hd, "fvit_unpad_heads_f32: bad arguments");
  const long long total = (long long)rows_src * cols_src;
  unpad_heads_kernel<<<grid_cap(total, 256, 16), 256, 0, (cudaStream_t)stream>>>(src, lds, dst, ldd, rows_src, cols_src,
                                                                                  hd, hdp, pad_rows, pad_cols, scalar);
  return post_launch("unpad_heads_kernel");
}

int fvit_attn_bias_bwd(const float* dbias, const float* bias, const int64_t* index, int32_t heads, int32_t S,
                       int32_t L, const float* scalar, float* dtable, void* stream) {
  FVIT_CHECK(dbias && bias && index && dtable && heads > 0 && S > 0 && L > 0, "fvit_attn_bias_bwd: bad arguments");
  const long long total = (long long)heads * L * L;
  attn_bias_bwd_kernel<<<grid_cap(total, 256, 8), 256, 0, (cudaStream_t)stream>>>(
      dbias, bias, (const long long*)index, heads, S, L, scalar, dtable);
  return post_launch("attn_bias_bwd_kernel");
}

int fvit_cpb_mlp_bwd(const float* coords, int32_t P, const float* w1, const float* hidden, const float* dout,
                     int32_t D, const float* scalar, float* dw0, float* db0, float* dw1, void* stream) {
  FVIT_CHECK(coords && w1 && hidden && dout && dw0 && db0 && dw1 && P > 0 && D > 0, "fvit_cpb_mlp_bwd: bad arguments");
  cpb_mlp_bwd_w1_kernel<<<D, 512, P * sizeof(float), (cudaStream_t)stream>>>(P, hidden, dout, D, scalar, dw1);
  int rc = post_launch("cpb_mlp_bwd_w1_kernel");
  if (rc) return rc;
  int splits = D >= 512 ? 8 : (D >= 128 ? 4 : 1);
  const size_t smem = ((size_t)(D + splits - 1) / splits + 1) * sizeof(float);
  cpb_mlp_bwd_kernel<<<dim3((unsigned)P, 4, (unsigned)splits), 128, smem, (cudaStream_t)stream>>>(coords, P, w1, hidden,
                                                                                                   dout, D, scalar, dw0, db0);
  return post_launch("cpb_mlp_bwd_kernel");
}

int fvit_pool_bn_bwd(const float* xs, int64_t ldx, const int32_t* rows, int32_t B, int32_t T, int32_t C,
                     const float* mean, const float* rstd, const float* w, const float* dpool, int64_t lddp,
                     float* s1, float* s2, const float* scalar, float* g, int64_t ldg, float* dw, float* dbeta,
                     void* stream) {
  FVIT_CHECK(xs && mean && rstd && w && dpool && s1 && s2 && g && dw && dbeta && B > 0 && T > 0 && C > 0,
             "fvit_pool_bn_bwd: bad arguments");
  FVIT_CUDA(cudaMemsetAsync(s1, 0, C * sizeof(float), (cudaStream_t)stream));
  FVIT_CUDA(cudaMemsetAsync(s2, 0, C * sizeof(float), (cudaStream_t)stream));
  dim3 grid((unsigned)(B < 64 ? B : 64), (unsigned)((C + 127) / 128));
  pool_bn_bwd_reduce_kernel<<<grid, 128, 0, (cudaStream_t)stream>>>(xs, ldx, rows, B, T, C, mean, rstd, dpool, lddp,
                                                                    s1, s2);
  int rc = post_launch("pool_bn_bwd_reduce_kernel");
  if (rc) return rc;
  const long long total = (long long)B * T * C;
  pool_bn_bwd_apply_kernel<<<grid_cap(total, 256, 8), 256, 0, (cudaStream_t)stream>>>(
      xs, ldx, rows, B, T, C, mean, rstd, w, dpool, lddp, s1, s2, scalar, g, ldg, dw, dbeta);
  return post_launch("pool_bn_bwd_apply_kernel");
}

int fvit_scatter_add_rows(const float* src, int64_t lds, float* dst, int64_t ldd, const int32_t* map, int32_t rows,
                          int32_t C, void* stream) {
  FVIT_CHECK(src && dst && map && rows > 0 && C % 4 == 0 && lds % 4 == 0 && ldd % 4 == 0,
             "fvit_scatter_add_rows: bad arguments");
  const long long total = (long long)rows * (C / 4);
  scatter_add_rows_kernel<<<grid_cap(total, 256, 16), 256, 0, (cudaStream_t)stream>>>(src, lds, dst, ldd, map, rows, C);
  return post_launch("scatter_add_rows_kernel");
}

int fvit_bn_bwd(const void* gin, int32_t g_is_f16, int64_t ldg, const int32_t* g_rows, const void* raw16, int64_t ldr,
                const int32_t* r_rows, int32_t nrows, int32_t C, const float* mean, const float* rstd, const float* w,
                const float* b, int32_t act, const float* colmul, float* s1, float* s2, const float* scalar, void* out16,
                int64_t ldo, const int32_t* o_rows, float* dw, float* db, const float* row_scale, void* stream) {
  FVIT_CHECK(gin && raw16 && mean && rstd && w && b && s1 && s2 && out16 && dw && db && nrows > 0 && C > 0,
             "fvit_bn_bwd: bad arguments");
  FVIT_CHECK(act == FVIT_ACT_NONE || act == FVIT_ACT_RELU, "fvit_bn_bwd: act must be NONE or RELU");
  FVIT_CUDA(cudaMemsetAsync(s1, 0, C * sizeof(float), (cudaStream_t)stream));
  FVIT_CUDA(cudaMemsetAsync(s2, 0, C * sizeof(float), (cudaStream_t)stream));
  const cudaStream_t st = (cudaStream_t)stream;
  const bool vec = C % 4 == 0 && ldg % 4 == 0 && ldr % 4 == 0 && ldo % 4 == 0 &&
                   (reinterpret_cast<uintptr_t>(gin) % 16 == 0) && (reinterpret_cast<uintptr_t>(raw16) % 8 == 0) &&
                   (reinterpret_cast<uintptr_t>(out16) % 8 == 0);
  const bool vec8 = vec && ldr % 8 == 0 && ldo % 8 == 0 && (g_is_f16 ? ldg % 8 == 0 : true) &&
                    (reinterpret_cast<uintptr_t>(raw16) % 16 == 0) && (reinterpret_cast<uintptr_t>(out16) % 16 == 0) &&
                    (reinterpret_cast<uintptr_t>(gin) % 16 == 0);
  if (vec8) {
    const int c8 = (C + 7) / 8;
    int vpr = 1;
    while (vpr < 64 && vpr < c8) vpr *= 2;
    const unsigned gy = (unsigned)((c8 + vpr - 1) / vpr);
    const int RL = 256 / vpr;
    long long gx = ((long long)num_sms() * 6 + gy - 1) / gy;
    const long long gx_max = ((long long)nrows + RL * BN8_ROWS - 1) / (RL * BN8_ROWS);
    if (gx > gx_max) gx = gx_max;
    if (gx < 1) gx = 1;
    dim3 grid((unsigned)gx, gy);
    const float inv = 1.f / (float)nrows;
    if (g_is_f16) {
      bn_bwd_reduce_v8_kernel<1><<<grid, 256, 0, st>>>(gin, ldg, g_rows, (const __half*)raw16, ldr, r_rows, nrows, C, vpr,
                                                       mean, rstd, w, b, act, colmul, s1, s2, row_scale);
      bn_bwd_apply_v8_kernel<1><<<grid, 256, 0, st>>>(gin, ldg, g_rows, (const __half*)raw16, ldr, r_rows, nrows, C, vpr,
                                                      inv, mean, rstd, w, b, act, colmul, s1, s2, scalar,
                                                      (__half*)out16, ldo, o_rows, dw, db, row_scale);
    } else {
      bn_bwd_reduce_v8_kernel<0><<<grid, 256, 0, st>>>(gin, ldg, g_rows, (const __half*)raw16, ldr, r_rows, nrows, C, vpr,
                                                       mean, rstd, w, b, act, colmul, s1, s2, row_scale);
      bn_bwd_apply_v8_kernel<0><<<grid, 256, 0, st>>>(gin, ldg, g_rows, (const __half*)raw16, ldr, r_rows, nrows, C, vpr,
                                                      inv, mean, rstd, w, b, act, colmul, s1, s2, scalar,
                                                      (__half*)out16, ldo, o_rows, dw, db, row_scale);
    }
    g_launches.fetch_add(1, std::memory_order_relaxed);
    return post_launch("bn_bwd v8 kernels");
  }
  if (vec) {
    int vpr = 1;
    while (vpr < 64 && vpr < C / 4) vpr *= 2;
    const unsigned gy = (unsigned)((C / 4 + vpr - 1) / vpr);
    const int RL = 256 / vpr;
    long long gx = ((long long)num_sms() * 8 + gy - 1) / gy;
    const long long gx_max = ((long long)nrows + RL * 4 - 1) / (RL * 4);
    if (gx > gx_max) gx = gx_max;
    if (gx < 1) gx = 1;
    dim3 grid((unsigned)gx, gy);
    const float inv = 1.f / (float)nrows;
    if (g_is_f16) {
      bn_bwd_reduce_v4_kernel<1><<<grid, 256, 0, st>>>(gin, ldg, g_rows, (const __half*)raw16, ldr, r_rows, nrows, C, vpr,
                                                       mean, rstd, w, b, act, colmul, s1, s2, row_scale);
      bn_bwd_apply_v4_kernel<1><<<grid, 256, 0, st>>>(gin, ldg, g_rows, (const __half*)raw16, ldr, r_rows, nrows, C, vpr,
                                                      inv, mean, rstd, w, b, act, colmul, s1, s2, scalar,
                                                      (__half*)out16, ldo, o_rows, dw, db, row_scale);
    } else {
      bn_bwd_reduce_v4_kernel<0><<<grid, 256, 0, st>>>(gin, ldg, g_rows, (const __half*)raw16, ldr, r_rows, nrows, C, vpr,
                                                       mean, rstd, w, b, act, colmul, s1, s2, row_scale);
      bn_bwd_apply_v4_kernel<0><<<grid, 256, 0, st>>>(gin, ldg, g_rows, (const __half*)raw16, ldr, r_rows, nrows, C, vpr,
                                                      inv, mean, rstd, w, b, act, colmul, s1, s2, scalar,
                                                      (__half*)out16, ldo, o_rows, dw, db, row_scale);
    }
    g_launches.fetch_add(1, std::memory_order_relaxed);
    return post_launch("bn_bwd v4 kernels");
  }
  dim3 grid((unsigned)grid_cap(((long long)nrows + 15) / 16, 1, 24), (unsigned)((C + 63) / 64));
  const long long total = (long long)nrows * C;
  const int g2 = grid_cap(total, 256, 16);
  if (g_is_f16) {
    bn_bwd_reduce_kernel<1><<<grid, 256, 0, (cudaStream_t)stream>>>(gin, ldg, g_rows, (const __half*)raw16, ldr, r_rows,
                                                                    nrows, C, mean, rstd, w, b, act, colmul, s1, s2, row_scale);
    bn_bwd_apply_kernel<1><<<g2, 256, 0, (cudaStream_t)stream>>>(gin, ldg, g_rows, (const __half*)raw16, ldr, r_rows,
                                                                 nrows, C, (float)nrows, mean, rstd, w, b, act, colmul, s1,
                                                                 s2, scalar, (__half*)out16, ldo, o_rows, dw, db, row_scale);
  } else {
    bn_bwd_reduce_kernel<0><<<grid, 256, 0, (cudaStream_t)stream>>>(gin, ldg, g_rows, (const __half*)raw16, ldr, r_rows,
                                                                    nrows, C, mean, rstd, w, b, act, colmul, s1, s2, row_scale);
    bn_bwd_apply_kernel<0><<<g2, 256, 0, (cudaStream_t)stream>>>(gin, ldg, g_rows, (const __half*)raw16, ldr, r_rows,
                                                                 nrows, C, (float)nrows, mean, rstd, w, b, act, colmul, s1,
                                                                 s2, scalar, (__half*)out16, ldo, o_rows, dw, db, row_scale);
  }
  g_launches.fetch_add(1, std::memory_order_relaxed);
  return post_launch("bn_bwd kernels");
}

int fvit_unpack_conv_grad(const float* src, int32_t ld_ci, float* dst, int32_t cout, int32_t cin, void* stream) {
  FVIT_CHECK(src && dst && cout > 0 && cin > 0 && ld_ci >= cin, "fvit_unpack_conv_grad: bad arguments");
  const long long total = (long long)cout * cin * 9;
  unpack_conv_grad_kernel<<<grid_cap(total, 256, 8), 256, 0, (cudaStream_t)stream>>>(src, ld_ci, dst, cout, cin);
  return post_launch("unpack_conv_grad_kernel");
}

}  // extern "C" (the launch templates below have C++ linkage)

// the input-gradient kernels of the TokenInitializer backward (fvit_token_init_bwd, fvit_token_init_dgrad)
template <bool kNchwTokens>
static int token_init_dx_launch(const float* g, int64_t ldg, const int32_t* pix_map, const int32_t* ct_row_map, int32_t B,
                                int32_t Hp, int32_t Wp, int32_t C, const float* w, int32_t kh, int32_t kw, int32_t sh,
                                int32_t sw, int32_t oh, int32_t ow, float* gx, int64_t ldgx, void* stream) {
  const size_t tile_smem = ((size_t)oh * ow + (size_t)Hp * Wp) * 32 * sizeof(float);
  if (tile_smem <= 48 * 1024 && B <= 65535) {  // the whole map of one image fits: pool backward formed once per pixel
    dim3 gt((unsigned)((C + 31) / 32), (unsigned)B);
    token_init_bwd_tile_kernel<kNchwTokens><<<gt, 256, tile_smem, (cudaStream_t)stream>>>(g, ldg, pix_map, ct_row_map, Hp, Wp, C, w, kh,
                                                                             kw, sh, sw, oh, ow, gx, ldgx);
    return post_launch("token_init_bwd_tile_kernel");
  }
  const int cb = C >= 256 ? 256 : (C >= 128 ? 128 : 64);
  const long long npos = (long long)B * Hp * Wp;
  dim3 gd((unsigned)((C + cb - 1) / cb), (unsigned)(npos < 65535 ? npos : 65535));
  token_init_bwd_kernel<kNchwTokens><<<gd, cb, 0, (cudaStream_t)stream>>>(g, ldg, pix_map, ct_row_map, B, Hp, Wp, C, w, kh, kw, sh, sw,
                                                             oh, ow, gx, ldgx);
  return post_launch("token_init_bwd_kernel");
}

template <bool kNchwTokens>
static int token_init_bwd_launch(const float* g, int64_t ldg, const void* x16, int64_t ldx, const int32_t* pix_map,
                                 const int32_t* ct_row_map, int32_t B, int32_t Hp, int32_t Wp, int32_t C, const float* w,
                                 int32_t kh, int32_t kw, int32_t sh, int32_t sw, int32_t oh, int32_t ow, const float* scalar,
                                 float* gx, int64_t ldgx, float* dw, float* dbias, void* stream) {
  FVIT_CHECK(g && x16 && pix_map && ct_row_map && w && gx && dw && dbias, "fvit_token_init_bwd: null argument");
  const int npos4 = (B * oh * ow + 3) / 4;
  dim3 gw((unsigned)((C + 127) / 128), (unsigned)(npos4 < 512 ? npos4 : 512));
  token_init_wgrad_kernel<kNchwTokens><<<gw, 512, 0, (cudaStream_t)stream>>>(g, ldg, (const __half*)x16, ldx, pix_map,
                                                                             ct_row_map, B, Hp, Wp, C, kh, kw, sh, sw, oh,
                                                                             ow, scalar, dw, dbias);
  int rc = post_launch("token_init_wgrad_kernel");
  if (rc) return rc;
  return token_init_dx_launch<kNchwTokens>(g, ldg, pix_map, ct_row_map, B, Hp, Wp, C, w, kh, kw, sh, sw, oh, ow, gx, ldgx,
                                           stream);
}

extern "C" {

int fvit_token_init_bwd(const float* g, int64_t ldg, const void* x16, int64_t ldx, const int32_t* pix_map,
                        const int32_t* ct_row_map, int32_t B, int32_t Hp, int32_t Wp, int32_t C, const float* w,
                        int32_t kh, int32_t kw, int32_t sh, int32_t sw, int32_t oh, int32_t ow, const float* scalar,
                        float* gx, int64_t ldgx, float* dw, float* dbias, void* stream) {
  return token_init_bwd_launch<false>(g, ldg, x16, ldx, pix_map, ct_row_map, B, Hp, Wp, C, w, kh, kw, sh, sw, oh, ow,
                                      scalar, gx, ldgx, dw, dbias, stream);
}

int fvit_token_init_nchw_bwd(const float* g, int64_t ldg, const void* x16, int64_t ldx, const int32_t* pix_map,
                             const int32_t* ct_row_map, int32_t B, int32_t Hp, int32_t Wp, int32_t C, const float* w,
                             int32_t kh, int32_t kw, int32_t sh, int32_t sw, int32_t oh, int32_t ow, const float* scalar,
                             float* gx, int64_t ldgx, float* dw, float* dbias, void* stream) {
  return token_init_bwd_launch<true>(g, ldg, x16, ldx, pix_map, ct_row_map, B, Hp, Wp, C, w, kh, kw, sh, sw, oh, ow,
                                     scalar, gx, ldgx, dw, dbias, stream);
}

int fvit_token_init_dgrad(const float* g, int64_t ldg, const int32_t* pix_map, const int32_t* ct_row_map, int32_t B,
                          int32_t Hp, int32_t Wp, int32_t C, const float* w, int32_t kh, int32_t kw, int32_t sh,
                          int32_t sw, int32_t oh, int32_t ow, float* gx, int64_t ldgx, void* stream) {
  FVIT_CHECK(g && pix_map && ct_row_map && w && gx && B > 0 && C > 0, "fvit_token_init_dgrad: bad arguments");
  return token_init_dx_launch<false>(g, ldg, pix_map, ct_row_map, B, Hp, Wp, C, w, kh, kw, sh, sw, oh, ow, gx, ldgx,
                                     stream);
}

int fvit_token_init_nchw_dgrad(const float* g, int64_t ldg, const int32_t* pix_map, const int32_t* ct_row_map, int32_t B,
                               int32_t Hp, int32_t Wp, int32_t C, const float* w, int32_t kh, int32_t kw, int32_t sh,
                               int32_t sw, int32_t oh, int32_t ow, float* gx, int64_t ldgx, void* stream) {
  FVIT_CHECK(g && pix_map && ct_row_map && w && gx && B > 0 && C > 0, "fvit_token_init_nchw_dgrad: bad arguments");
  return token_init_dx_launch<true>(g, ldg, pix_map, ct_row_map, B, Hp, Wp, C, w, kh, kw, sh, sw, oh, ow, gx, ldgx,
                                    stream);
}

int fvit_propagate_bwd(float* g, int64_t ldg, const float* xs, int64_t ldx, const int32_t* src_map, int32_t rows, int32_t C,
                       const float* gamma, const float* scalar, float* dgamma, void* stream) {
  FVIT_CHECK(g && xs && src_map && rows > 0 && C > 0, "fvit_propagate_bwd: bad arguments");
  dim3 grid((unsigned)grid_cap(((long long)rows + 3) / 4, 1, 4), (unsigned)((C + 63) / 64));
  propagate_bwd_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(g, ldg, xs, ldx, src_map, rows, C, gamma, scalar, dgamma);
  return post_launch("propagate_bwd_kernel");
}

}  // extern "C"
