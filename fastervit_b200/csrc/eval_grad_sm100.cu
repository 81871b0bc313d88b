// Backward kernels of an eval()-mode forward (include/fvit.h "Eval-mode gradients"): BatchNorm2d on running
// statistics, the head's running-statistics BatchNorm folded into the average pool, and the image gradient of the
// stem's first convolution. All three are HBM-bound single passes.
#include <cuda_fp16.h>

#include "../../include/fvit.h"
#include "common.h"

namespace fvit {

// ---------------------------------------------------------------------------------- BatchNorm2d, running statistics
// xhat = (raw - mean) * rstd with rstd = rsqrt(var + eps) fixed, so the backward has no mean(dy) / xhat*mean(dy*xhat)
// terms: out16 = w*rstd*dy, dw += scalar * sum dy*xhat, db += scalar * sum dy, dy = gin * colmul masked by ReLU'.
// 8-channel version (16-byte fp16 rows / 2 x float4 fp32 rows): a lane owns 8 channels of a row, vpr lanes cover a
// row, 256 / vpr rows per block pass; per-block partial sums, one set of atomics per block.
constexpr int BNE_ROWS = 4;  // rows per trip (fp16 gin; 2 for fp32): all index loads, then all data loads, then the math
template <int G16>
__global__ void __launch_bounds__(256, 2)
bn_eval_bwd_v8_kernel(const void* __restrict__ gin, long long ldg, const int* __restrict__ g_rows,
                      const __half* __restrict__ raw, long long ldr, const int* __restrict__ r_rows, int nrows, int C,
                      int vpr, const float* __restrict__ mean, const float* __restrict__ var, float eps,
                      const float* __restrict__ w, const float* __restrict__ b, int act,
                      const float* __restrict__ colmul, const float* __restrict__ scalar, __half* __restrict__ out,
                      long long ldo, const int* __restrict__ o_rows, float* __restrict__ dw, float* __restrict__ db) {
  __shared__ float red[2][8][257];
  const int cx = threadIdx.x % vpr, rl = threadIdx.x / vpr, RL = 256 / vpr;
  const int c = (blockIdx.y * vpr + cx) * 8;
  const int nv = min(8, C - c);
  constexpr int R = G16 ? BNE_ROWS : BNE_ROWS / 2;   // (an fp32 row chunk takes twice the registers)
  float a1[8], a2[8];
#pragma unroll
  for (int u = 0; u < 8; ++u) a1[u] = a2[u] = 0.f;
  if (nv > 0) {
    // xhat = raw*rs + nm ; pre-activation xhat*wc + bc ; out = kk*dy (kk = 0 on padding columns)
    float rs[8], nm[8], wc[8], bc[8], kk[8];
#pragma unroll
    for (int u = 0; u < 8; ++u) {
      const bool in = u < nv;
      rs[u] = in ? rsqrtf(__ldg(var + c + u) + eps) : 0.f;
      nm[u] = in ? -__ldg(mean + c + u) * rs[u] : 0.f;
      wc[u] = in ? __ldg(w + c + u) : 0.f;
      bc[u] = in ? __ldg(b + c + u) : 0.f;
      kk[u] = wc[u] * rs[u] * (in && colmul ? __ldg(colmul + c + u) : 1.f);
    }
    const bool relu = act == FVIT_ACT_RELU;
    const bool same_rows = g_rows == r_rows, same_out = o_rows == g_rows;
    const int rstep = gridDim.x * RL;
    for (int r0 = blockIdx.x * RL + rl; r0 < nrows; r0 += R * rstep) {
      long long rg[R], rr[R], ro[R];
#pragma unroll
      for (int t = 0; t < R; ++t) {
        const int r = r0 + t * rstep;
        const bool ok = r < nrows;
        rg[t] = ok ? (g_rows ? (long long)g_rows[r] : (long long)r) : -1;
        rr[t] = same_rows ? rg[t] : (ok ? (r_rows ? (long long)r_rows[r] : (long long)r) : -1);
        ro[t] = same_out ? rg[t] : (ok ? (o_rows ? (long long)o_rows[r] : (long long)r) : -1);
      }
      uint4 ga[R], gb[R], xp[R];
#pragma unroll
      for (int t = 0; t < R; ++t) {
        ga[t] = gb[t] = xp[t] = make_uint4(0u, 0u, 0u, 0u);
        if (rg[t] >= 0) {
          if (G16) {
            ga[t] = *reinterpret_cast<const uint4*>(reinterpret_cast<const __half*>(gin) + rg[t] * ldg + c);
          } else {
            const uint4* p4 = reinterpret_cast<const uint4*>(reinterpret_cast<const float*>(gin) + rg[t] * ldg + c);
            ga[t] = p4[0];
            if (nv > 4) gb[t] = p4[1];
          }
          xp[t] = *reinterpret_cast<const uint4*>(raw + rr[t] * ldr + c);
        }
      }
#pragma unroll
      for (int t = 0; t < R; ++t) {
        if (rg[t] < 0) continue;
        float dy[8], xt[8];
        if (G16) {
          const __half2* h = reinterpret_cast<const __half2*>(&ga[t]);
#pragma unroll
          for (int u = 0; u < 4; ++u) dy[2 * u] = __low2float(h[u]), dy[2 * u + 1] = __high2float(h[u]);
        } else {
          dy[0] = __uint_as_float(ga[t].x), dy[1] = __uint_as_float(ga[t].y);
          dy[2] = __uint_as_float(ga[t].z), dy[3] = __uint_as_float(ga[t].w);
          dy[4] = __uint_as_float(gb[t].x), dy[5] = __uint_as_float(gb[t].y);
          dy[6] = __uint_as_float(gb[t].z), dy[7] = __uint_as_float(gb[t].w);
        }
        const __half2* hx = reinterpret_cast<const __half2*>(&xp[t]);
#pragma unroll
        for (int u = 0; u < 4; ++u) xt[2 * u] = __low2float(hx[u]), xt[2 * u + 1] = __high2float(hx[u]);
        __half2 h[4];
#pragma unroll
        for (int u = 0; u < 8; u += 2) {
          float o[2];
#pragma unroll
          for (int v = 0; v < 2; ++v) {
            const float xh = fmaf(xt[u + v], rs[u + v], nm[u + v]);
            float d = u + v < nv ? dy[u + v] : 0.f;
            if (relu && fmaf(xh, wc[u + v], bc[u + v]) <= 0.f) d = 0.f;
            o[v] = kk[u + v] * d;   // (colmul folded into kk and, below, into the sums' factor)
            a1[u + v] += d;
            a2[u + v] = fmaf(d, xh, a2[u + v]);
          }
          h[u / 2] = __floats2half2_rn(o[0], o[1]);
        }
        *reinterpret_cast<uint4*>(out + ro[t] * ldo + c) = *reinterpret_cast<const uint4*>(h);
      }
    }
  }
#pragma unroll
  for (int u = 0; u < 8; ++u) red[0][u][threadIdx.x] = a1[u], red[1][u][threadIdx.x] = a2[u];
  __syncthreads();
  const float sc = scalar ? __ldg(scalar) : 1.f;
  for (int q = threadIdx.x; q < 16 * vpr; q += 256) {
    const int which = q / (8 * vpr), u = (q / vpr) & 7, lane = q % vpr;
    const int cc = (blockIdx.y * vpr + lane) * 8 + u;
    if (cc < C) {
      float t = 0.f;
      for (int k = 0; k < RL; ++k) t += red[which][u][k * vpr + lane];
      t *= sc * (colmul ? __ldg(colmul + cc) : 1.f);
      atomicAdd((which ? dw : db) + cc, t);
    }
  }
}

// Any layout: block = 64 columns x 4 row lanes.
template <int G16>
__global__ void __launch_bounds__(256)
bn_eval_bwd_kernel(const void* __restrict__ gin, long long ldg, const int* __restrict__ g_rows,
                   const __half* __restrict__ raw, long long ldr, const int* __restrict__ r_rows, int nrows, int C,
                   const float* __restrict__ mean, const float* __restrict__ var, float eps,
                   const float* __restrict__ w, const float* __restrict__ b, int act,
                   const float* __restrict__ colmul, const float* __restrict__ scalar, __half* __restrict__ out,
                   long long ldo, const int* __restrict__ o_rows, float* __restrict__ dw, float* __restrict__ db) {
  __shared__ float red[2][4][64];
  const int c = blockIdx.y * 64 + (threadIdx.x & 63);
  const int rl = threadIdx.x >> 6;
  float a1 = 0.f, a2 = 0.f;
  if (c < C) {
    const float rs = rsqrtf(var[c] + eps), mu = mean[c], wc = w[c], bc = b[c], cm = colmul ? colmul[c] : 1.f;
    for (int r = blockIdx.x * 4 + rl; r < nrows; r += gridDim.x * 4) {
      const long long rg = g_rows ? g_rows[r] : r, rr = r_rows ? r_rows[r] : r, ro = o_rows ? o_rows[r] : r;
      float dy = G16 ? __half2float(reinterpret_cast<const __half*>(gin)[rg * ldg + c])
                     : reinterpret_cast<const float*>(gin)[rg * ldg + c];
      const float xh = (__half2float(raw[rr * ldr + c]) - mu) * rs;
      if (act == FVIT_ACT_RELU && fmaf(xh, wc, bc) <= 0.f) dy = 0.f;
      out[ro * ldo + c] = __float2half_rn(wc * rs * cm * dy);
      a1 += dy;
      a2 += dy * xh;
    }
  }
  red[0][rl][threadIdx.x & 63] = a1;
  red[1][rl][threadIdx.x & 63] = a2;
  __syncthreads();
  if (rl == 0 && c < C) {
    const int k = threadIdx.x & 63;
    const float sc = (scalar ? __ldg(scalar) : 1.f) * (colmul ? colmul[c] : 1.f);
    atomicAdd(db + c, sc * (red[0][0][k] + red[0][1][k] + red[0][2][k] + red[0][3][k]));
    atomicAdd(dw + c, sc * (red[1][0][k] + red[1][1][k] + red[1][2][k] + red[1][3][k]));
  }
}

// ---------------------------------------------------------------------------------- BatchNorm2d, data gradient only
// The same backward when nobody wants dw / db (a stage whose parameters get no gradient): out16 = k * dy with
// k[c] = scale[c] * colmul[c] * *scalar, scale = w * rsqrt(var + eps) as the forward folded it, masked by ReLU'
// (sign of raw * scale + shift, the forward's own pre-activation). No xhat, no sums, no atomics: raw is read only for
// the mask, so without an activation the pass moves dy in and dz out and nothing else.
// Layout as bn_eval_bwd_v8_kernel: a lane owns 8 channels, vpr lanes cover a row, R rows in flight per thread.
template <int G16, int RELU>
__global__ void __launch_bounds__(256, 3)
bn_eval_dgrad_v8_kernel(const void* __restrict__ gin, long long ldg, const int* __restrict__ g_rows,
                        const __half* __restrict__ raw, long long ldr, const int* __restrict__ r_rows, int nrows, int C,
                        int vpr, const float* __restrict__ scale, const float* __restrict__ shift,
                        const float* __restrict__ colmul, const float* __restrict__ scalar, __half* __restrict__ out,
                        long long ldo, const int* __restrict__ o_rows) {
  const int cx = threadIdx.x % vpr, rl = threadIdx.x / vpr, RL = 256 / vpr;
  const int c = (blockIdx.y * vpr + cx) * 8;
  const int nv = min(8, C - c);
  if (nv <= 0) return;
  constexpr int R = G16 ? BNE_ROWS : BNE_ROWS / 2;
  const float s = scalar ? __ldg(scalar) : 1.f;
  float sc[8], sh[8], kk[8];
#pragma unroll
  for (int u = 0; u < 8; ++u) {
    const bool in = u < nv;
    sc[u] = in ? __ldg(scale + c + u) : 0.f;
    sh[u] = in && RELU ? __ldg(shift + c + u) : 0.f;
    kk[u] = sc[u] * s * (in && colmul ? __ldg(colmul + c + u) : 1.f);
  }
  const bool same_rows = g_rows == r_rows, same_out = o_rows == g_rows;
  const int rstep = gridDim.x * RL;
  for (int r0 = blockIdx.x * RL + rl; r0 < nrows; r0 += R * rstep) {
    long long rg[R], rr[R], ro[R];
#pragma unroll
    for (int t = 0; t < R; ++t) {
      const int r = r0 + t * rstep;
      const bool ok = r < nrows;
      rg[t] = ok ? (g_rows ? (long long)g_rows[r] : (long long)r) : -1;
      rr[t] = !RELU || same_rows ? rg[t] : (ok ? (r_rows ? (long long)r_rows[r] : (long long)r) : -1);
      ro[t] = same_out ? rg[t] : (ok ? (o_rows ? (long long)o_rows[r] : (long long)r) : -1);
      if (ro[t] < 0 || rr[t] < 0) rg[t] = -1;   // (a row any of the maps drops is skipped)
    }
    uint4 ga[R], gb[R], xp[R];
#pragma unroll
    for (int t = 0; t < R; ++t) {
      ga[t] = gb[t] = xp[t] = make_uint4(0u, 0u, 0u, 0u);
      if (rg[t] >= 0) {
        if (G16) {
          ga[t] = *reinterpret_cast<const uint4*>(reinterpret_cast<const __half*>(gin) + rg[t] * ldg + c);
        } else {
          const uint4* p4 = reinterpret_cast<const uint4*>(reinterpret_cast<const float*>(gin) + rg[t] * ldg + c);
          ga[t] = p4[0];
          if (nv > 4) gb[t] = p4[1];
        }
        if (RELU) xp[t] = *reinterpret_cast<const uint4*>(raw + rr[t] * ldr + c);
      }
    }
#pragma unroll
    for (int t = 0; t < R; ++t) {
      if (rg[t] < 0) continue;
      float dy[8];
      if (G16) {
        const __half2* h = reinterpret_cast<const __half2*>(&ga[t]);
#pragma unroll
        for (int u = 0; u < 4; ++u) dy[2 * u] = __low2float(h[u]), dy[2 * u + 1] = __high2float(h[u]);
      } else {
        dy[0] = __uint_as_float(ga[t].x), dy[1] = __uint_as_float(ga[t].y);
        dy[2] = __uint_as_float(ga[t].z), dy[3] = __uint_as_float(ga[t].w);
        dy[4] = __uint_as_float(gb[t].x), dy[5] = __uint_as_float(gb[t].y);
        dy[6] = __uint_as_float(gb[t].z), dy[7] = __uint_as_float(gb[t].w);
      }
      const __half2* hx = reinterpret_cast<const __half2*>(&xp[t]);
      __half2 h[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        float o0 = kk[2 * u] * dy[2 * u], o1 = kk[2 * u + 1] * dy[2 * u + 1];   // (kk = 0 on padding columns)
        if (RELU) {
          if (fmaf(__low2float(hx[u]), sc[2 * u], sh[2 * u]) <= 0.f) o0 = 0.f;
          if (fmaf(__high2float(hx[u]), sc[2 * u + 1], sh[2 * u + 1]) <= 0.f) o1 = 0.f;
        }
        h[u] = __floats2half2_rn(o0, o1);
      }
      *reinterpret_cast<uint4*>(out + ro[t] * ldo + c) = *reinterpret_cast<const uint4*>(h);
    }
  }
}

// Any layout: one thread per element.
template <int G16>
__global__ void __launch_bounds__(256)
bn_eval_dgrad_kernel(const void* __restrict__ gin, long long ldg, const int* __restrict__ g_rows,
                     const __half* __restrict__ raw, long long ldr, const int* __restrict__ r_rows, int nrows, int C,
                     const float* __restrict__ scale, const float* __restrict__ shift, int relu,
                     const float* __restrict__ colmul, const float* __restrict__ scalar, __half* __restrict__ out,
                     long long ldo, const int* __restrict__ o_rows) {
  const float s = scalar ? __ldg(scalar) : 1.f;
  const long long total = (long long)nrows * C;
  for (long long i = blockIdx.x * 256LL + threadIdx.x; i < total; i += (long long)gridDim.x * 256) {
    const int r = (int)(i / C), c = (int)(i % C);
    const long long rg = g_rows ? g_rows[r] : r, rr = r_rows ? r_rows[r] : r, ro = o_rows ? o_rows[r] : r;
    if (rg < 0 || ro < 0 || (relu && rr < 0)) continue;
    float dy = G16 ? __half2float(reinterpret_cast<const __half*>(gin)[rg * ldg + c])
                   : reinterpret_cast<const float*>(gin)[rg * ldg + c];
    const float sc = scale[c];
    if (relu && fmaf(__half2float(raw[rr * ldr + c]), sc, shift[c]) <= 0.f) dy = 0.f;
    out[ro * ldo + c] = __float2half_rn(sc * s * (colmul ? colmul[c] : 1.f) * dy);
  }
}

// ---------------------------------------------------------------------------------- head: running-statistics BN + pool
// pooled[b,c] = mean_t (xhat[b,t,c]*w + beta): g[row(b,t)][c] = dpool[b,c]/T * w*rstd (the same for every t),
// dw += scalar * sum_b dpool * mean_t xhat, dbeta += scalar * sum_b dpool. Block = 128 columns; blocks stride over b.
__global__ void __launch_bounds__(128)
pool_bn_eval_bwd_kernel(const float* __restrict__ xs, long long ldx, const int* __restrict__ rows, int B, int T, int C,
                        const float* __restrict__ mean, const float* __restrict__ var, float eps,
                        const float* __restrict__ w, const float* __restrict__ dpool, long long lddp,
                        const float* __restrict__ scalar, float* __restrict__ g, long long ldg, float* __restrict__ dw,
                        float* __restrict__ dbeta) {
  const int c = blockIdx.y * blockDim.x + threadIdx.x;
  if (c >= C) return;
  const float mu = mean[c], rs = rsqrtf(var[c] + eps), k = w[c] * rs / (float)T;
  float a1 = 0.f, a2 = 0.f;
  for (int b = blockIdx.x; b < B; b += gridDim.x) {
    const float d = dpool[(long long)b * lddp + c];
    const float gv = d * k;
    const int* rb = rows ? rows + (long long)b * T : nullptr;
    float sx = 0.f;
#pragma unroll 4
    for (int t = 0; t < T; ++t) {
      const long long row = rb ? (long long)rb[t] : (long long)b * T + t;
      sx += xs[row * ldx + c] - mu;
      g[row * ldg + c] = gv;
    }
    a1 += d;
    a2 = fmaf(d, sx * rs / (float)T, a2);
  }
  const float sc = scalar ? __ldg(scalar) : 1.f;
  atomicAdd(dw + c, a2 * sc);
  atomicAdd(dbeta + c, a1 * sc);
}

// ---------------------------------------------------------------------------------- stem image gradient
// dx[b][ci][y][x] = scalar * sum_{co, ky, kx : y = 2 oy - 1 + ky, x = 2 ox - 1 + kx} w[co][ci][ky][kx] * dz[b,oy,ox][co]
// (3x3, stride 2, pad 1, 3 input channels). A block owns 15 x 15 output positions and the 30 x 30 input pixels that
// read them; it forms the 27 tap products P[pos][ci][ky][kx] = sum_co w * dz of a 16 x 16 window (one halo row and
// column: an odd input coordinate also reads the next output position) in shared memory, then every pixel gathers
// its 1, 2 or 4 entries -- no atomics, so the result is deterministic.
constexpr int SD_OWN = 15, SD_WIN = 16;
__global__ void __launch_bounds__(256)
stem_conv_dgrad_kernel(const __half* __restrict__ dz, long long lddz, int vec, int H, int W, int H1, int W1,
                       const float* __restrict__ wgt, int cout, const float* __restrict__ scalar,
                       float* __restrict__ dx) {
  extern __shared__ float4 smem4[];
  float* wsm = reinterpret_cast<float*>(smem4);   // [cout][28]: w[co][ci*9 + ky*3 + kx], zero padded
  float* P = wsm + cout * 28;                    // [256][27]
  const int b = blockIdx.z, oy0 = blockIdx.y * SD_OWN, ox0 = blockIdx.x * SD_OWN;
  for (int i = threadIdx.x; i < cout * 28; i += 256) {
    const int co = i / 28, k = i % 28;
    wsm[i] = k < 27 ? wgt[co * 27 + k] : 0.f;
  }
  __syncthreads();
  const int oy = oy0 + threadIdx.x / SD_WIN, ox = ox0 + threadIdx.x % SD_WIN;
  float acc[28];
#pragma unroll
  for (int k = 0; k < 28; ++k) acc[k] = 0.f;
  if (oy < H1 && ox < W1) {
    const __half* row = dz + ((long long)(b * H1 + oy) * W1 + ox) * lddz;
    int co = 0;
    if (vec) {
      for (; co + 8 <= cout; co += 8) {
        const uint4 pk = *reinterpret_cast<const uint4*>(row + co);
        const __half2* h = reinterpret_cast<const __half2*>(&pk);
        float d[8];
#pragma unroll
        for (int u = 0; u < 4; ++u) d[2 * u] = __low2float(h[u]), d[2 * u + 1] = __high2float(h[u]);
#pragma unroll
        for (int u = 0; u < 8; ++u) {
          const float4* wr = reinterpret_cast<const float4*>(wsm + (co + u) * 28);
#pragma unroll
          for (int q = 0; q < 7; ++q) {
            const float4 wv = wr[q];
            acc[4 * q] = fmaf(d[u], wv.x, acc[4 * q]);
            acc[4 * q + 1] = fmaf(d[u], wv.y, acc[4 * q + 1]);
            acc[4 * q + 2] = fmaf(d[u], wv.z, acc[4 * q + 2]);
            acc[4 * q + 3] = fmaf(d[u], wv.w, acc[4 * q + 3]);
          }
        }
      }
    }
    for (; co < cout; ++co) {
      const float d = __half2float(row[co]);
#pragma unroll
      for (int k = 0; k < 27; ++k) acc[k] = fmaf(d, wsm[co * 28 + k], acc[k]);
    }
  }
  // (positions outside the map keep P = 0, so the gather below needs no bounds test on them)
#pragma unroll
  for (int k = 0; k < 27; ++k) P[threadIdx.x * 27 + k] = acc[k];
  __syncthreads();
  const float s = __ldg(scalar);
  constexpr int SPAN = 2 * SD_OWN;
  for (int i = threadIdx.x; i < 3 * SPAN * SPAN; i += 256) {
    const int ci = i / (SPAN * SPAN), yy = (i / SPAN) % SPAN, xx = i % SPAN;
    const int y = 2 * oy0 + yy, x = 2 * ox0 + xx;
    if (y >= H || x >= W) continue;
    // even coordinate: tap 1 of output position c/2; odd: tap 0 of (c+1)/2 and tap 2 of (c-1)/2
    const int nky = (yy & 1) ? 2 : 1, nkx = (xx & 1) ? 2 : 1;
    float v = 0.f;
    for (int a = 0; a < nky; ++a) {
      const int ky = (yy & 1) ? 2 * a : 1, ly = (yy & 1) ? (yy + 1) / 2 - a : yy / 2;
      for (int e = 0; e < nkx; ++e) {
        const int kx = (xx & 1) ? 2 * e : 1, lx = (xx & 1) ? (xx + 1) / 2 - e : xx / 2;
        v += P[(ly * SD_WIN + lx) * 27 + ci * 9 + ky * 3 + kx];
      }
    }
    dx[(((long long)b * 3 + ci) * H + y) * W + x] = v * s;
  }
}

// col2im of the same convolution for any channel count: the tap products arrive precomputed as fp32 rows
// dcol[(b*H1 + oy)*W1 + ox][ci*9 + ky*3 + kx] (the GEMM dz . W1), and dx gathers them exactly as above. A block owns
// the same 15 x 15 positions / 30 x 30 pixels and walks the channels in chunks of SC_CH, staging each chunk's 16 x 16
// window of tap entries in shared memory, so the tile does not grow with cin.
constexpr int SC_CH = 4;
__global__ void __launch_bounds__(256)
stem_col2im_kernel(const float* __restrict__ dcol, long long ldc, int cin, int H, int W, int H1, int W1,
                   float* __restrict__ dx) {
  __shared__ float P[SD_WIN * SD_WIN * SC_CH * 9];   // [position][ci - c0][ky][kx]
  const int b = blockIdx.z, oy0 = blockIdx.y * SD_OWN, ox0 = blockIdx.x * SD_OWN;
  constexpr int SPAN = 2 * SD_OWN;
  for (int c0 = 0; c0 < cin; c0 += SC_CH) {
    const int nc = min(SC_CH, cin - c0), cols = nc * 9;
    // positions outside the map stage zeros, so the gather below needs no bounds test on them
    for (int i = threadIdx.x; i < SD_WIN * SD_WIN * cols; i += 256) {
      const int pos = i / cols, k = i - pos * cols;
      const int oy = oy0 + pos / SD_WIN, ox = ox0 + pos % SD_WIN;
      P[i] = (oy < H1 && ox < W1) ? __ldg(dcol + ((long long)(b * H1 + oy) * W1 + ox) * ldc + c0 * 9 + k) : 0.f;
    }
    __syncthreads();
    for (int i = threadIdx.x; i < nc * SPAN * SPAN; i += 256) {
      const int cl = i / (SPAN * SPAN), yy = (i / SPAN) % SPAN, xx = i % SPAN;
      const int y = 2 * oy0 + yy, x = 2 * ox0 + xx;
      if (y >= H || x >= W) continue;
      // even coordinate: tap 1 of output position c/2; odd: tap 0 of (c+1)/2 and tap 2 of (c-1)/2
      const int nky = (yy & 1) ? 2 : 1, nkx = (xx & 1) ? 2 : 1;
      float v = 0.f;
      for (int a = 0; a < nky; ++a) {
        const int ky = (yy & 1) ? 2 * a : 1, ly = (yy & 1) ? (yy + 1) / 2 - a : yy / 2;
        for (int e = 0; e < nkx; ++e) {
          const int kx = (xx & 1) ? 2 * e : 1, lx = (xx & 1) ? (xx + 1) / 2 - e : xx / 2;
          v += P[(ly * SD_WIN + lx) * cols + cl * 9 + ky * 3 + kx];
        }
      }
      dx[(((long long)b * cin + c0 + cl) * H + y) * W + x] = v;
    }
    __syncthreads();
  }
}

}  // namespace fvit

using namespace fvit;

extern "C" {

int fvit_bn_eval_bwd(const void* gin, int32_t g_is_f16, int64_t ldg, const int32_t* g_rows, const void* raw16,
                     int64_t ldr, const int32_t* r_rows, int32_t nrows, int32_t C, const float* mean, const float* var,
                     float eps, const float* w, const float* b, int32_t act, const float* colmul, const float* scalar,
                     void* out16, int64_t ldo, const int32_t* o_rows, float* dw, float* db, void* stream) {
  FVIT_CHECK(gin && raw16 && mean && var && w && b && out16 && dw && db && nrows > 0 && C > 0,
             "fvit_bn_eval_bwd: bad arguments");
  FVIT_CHECK(act == FVIT_ACT_NONE || act == FVIT_ACT_RELU, "fvit_bn_eval_bwd: act must be NONE or RELU");
  const cudaStream_t st = (cudaStream_t)stream;
  const bool vec8 = C % 4 == 0 && ldg % (g_is_f16 ? 8 : 4) == 0 && ldr % 8 == 0 && ldo % 8 == 0 &&
                    reinterpret_cast<uintptr_t>(gin) % 16 == 0 && reinterpret_cast<uintptr_t>(raw16) % 16 == 0 &&
                    reinterpret_cast<uintptr_t>(out16) % 16 == 0;
  if (vec8) {
    const int c8 = (C + 7) / 8;
    int vpr = 1;
    while (vpr < 64 && vpr < c8) vpr *= 2;
    const unsigned gy = (unsigned)((c8 + vpr - 1) / vpr);
    const int RL = 256 / vpr;
    long long gx = ((long long)num_sms() * 4 + gy - 1) / gy;
    const long long gx_max = ((long long)nrows + RL * BNE_ROWS - 1) / (RL * BNE_ROWS);
    if (gx > gx_max) gx = gx_max;
    if (gx < 1) gx = 1;
    dim3 grid((unsigned)gx, gy);
    if (g_is_f16)
      bn_eval_bwd_v8_kernel<1><<<grid, 256, 0, st>>>(gin, ldg, g_rows, (const __half*)raw16, ldr, r_rows, nrows, C, vpr,
                                                     mean, var, eps, w, b, act, colmul, scalar, (__half*)out16, ldo,
                                                     o_rows, dw, db);
    else
      bn_eval_bwd_v8_kernel<0><<<grid, 256, 0, st>>>(gin, ldg, g_rows, (const __half*)raw16, ldr, r_rows, nrows, C, vpr,
                                                     mean, var, eps, w, b, act, colmul, scalar, (__half*)out16, ldo,
                                                     o_rows, dw, db);
    return post_launch("bn_eval_bwd_v8_kernel");
  }
  const unsigned gy = (unsigned)((C + 63) / 64);
  long long gx = ((long long)num_sms() * 8 + gy - 1) / gy;
  const long long gx_max = ((long long)nrows + 15) / 16;
  if (gx > gx_max) gx = gx_max;
  if (gx < 1) gx = 1;
  dim3 grid((unsigned)gx, gy);
  if (g_is_f16)
    bn_eval_bwd_kernel<1><<<grid, 256, 0, st>>>(gin, ldg, g_rows, (const __half*)raw16, ldr, r_rows, nrows, C, mean, var,
                                                eps, w, b, act, colmul, scalar, (__half*)out16, ldo, o_rows, dw, db);
  else
    bn_eval_bwd_kernel<0><<<grid, 256, 0, st>>>(gin, ldg, g_rows, (const __half*)raw16, ldr, r_rows, nrows, C, mean, var,
                                                eps, w, b, act, colmul, scalar, (__half*)out16, ldo, o_rows, dw, db);
  return post_launch("bn_eval_bwd_kernel");
}

int fvit_bn_eval_dgrad(const void* gin, int32_t g_is_f16, int64_t ldg, const int32_t* g_rows, const void* raw16,
                       int64_t ldr, const int32_t* r_rows, int32_t nrows, int32_t C, const float* scale,
                       const float* shift, int32_t act, const float* colmul, const float* scalar, void* out16,
                       int64_t ldo, const int32_t* o_rows, void* stream) {
  FVIT_CHECK(gin && scale && out16 && nrows > 0 && C > 0, "fvit_bn_eval_dgrad: bad arguments");
  FVIT_CHECK(act == FVIT_ACT_NONE || act == FVIT_ACT_RELU, "fvit_bn_eval_dgrad: act must be NONE or RELU");
  const bool relu = act == FVIT_ACT_RELU;
  FVIT_CHECK(!relu || (raw16 && shift), "fvit_bn_eval_dgrad: the ReLU mask needs raw16 and shift");
  const cudaStream_t st = (cudaStream_t)stream;
  const bool vec8 = C % 4 == 0 && ldg % (g_is_f16 ? 8 : 4) == 0 && (!relu || ldr % 8 == 0) && ldo % 8 == 0 &&
                    reinterpret_cast<uintptr_t>(gin) % 16 == 0 && (!relu || reinterpret_cast<uintptr_t>(raw16) % 16 == 0) &&
                    reinterpret_cast<uintptr_t>(out16) % 16 == 0;
  if (vec8) {
    const int c8 = (C + 7) / 8;
    int vpr = 1;
    while (vpr < 64 && vpr < c8) vpr *= 2;
    const unsigned gy = (unsigned)((c8 + vpr - 1) / vpr);
    const int RL = 256 / vpr;
    long long gx = ((long long)num_sms() * 8 + gy - 1) / gy;
    const long long gx_max = ((long long)nrows + RL * BNE_ROWS - 1) / (RL * BNE_ROWS);
    if (gx > gx_max) gx = gx_max;
    if (gx < 1) gx = 1;
    dim3 grid((unsigned)gx, gy);
#define FVIT_BN_DGRAD(G, R)                                                                                        \
  bn_eval_dgrad_v8_kernel<G, R><<<grid, 256, 0, st>>>(gin, ldg, g_rows, (const __half*)raw16, ldr, r_rows, nrows, C, \
                                                      vpr, scale, shift, colmul, scalar, (__half*)out16, ldo, o_rows)
    if (g_is_f16) {
      if (relu) FVIT_BN_DGRAD(1, 1); else FVIT_BN_DGRAD(1, 0);
    } else {
      if (relu) FVIT_BN_DGRAD(0, 1); else FVIT_BN_DGRAD(0, 0);
    }
#undef FVIT_BN_DGRAD
    return post_launch("bn_eval_dgrad_v8_kernel");
  }
  long long gx = ((long long)nrows * C + 255) / 256;
  const long long cap = (long long)num_sms() * 16;
  if (gx > cap) gx = cap;
  if (g_is_f16)
    bn_eval_dgrad_kernel<1><<<(unsigned)gx, 256, 0, st>>>(gin, ldg, g_rows, (const __half*)raw16, ldr, r_rows, nrows, C,
                                                          scale, shift, relu, colmul, scalar, (__half*)out16, ldo, o_rows);
  else
    bn_eval_dgrad_kernel<0><<<(unsigned)gx, 256, 0, st>>>(gin, ldg, g_rows, (const __half*)raw16, ldr, r_rows, nrows, C,
                                                          scale, shift, relu, colmul, scalar, (__half*)out16, ldo, o_rows);
  return post_launch("bn_eval_dgrad_kernel");
}

int fvit_pool_bn_eval_bwd(const float* xs, int64_t ldx, const int32_t* rows, int32_t B, int32_t T, int32_t C,
                          const float* mean, const float* var, float eps, const float* w, const float* dpool,
                          int64_t lddp, const float* scalar, float* g, int64_t ldg, float* dw, float* dbeta,
                          void* stream) {
  FVIT_CHECK(xs && mean && var && w && dpool && g && dw && dbeta && B > 0 && T > 0 && C > 0,
             "fvit_pool_bn_eval_bwd: bad arguments");
  const unsigned gy = (unsigned)((C + 127) / 128);
  long long gx = ((long long)num_sms() * 8 + gy - 1) / gy;
  if (gx > B) gx = B;
  pool_bn_eval_bwd_kernel<<<dim3((unsigned)gx, gy), 128, 0, (cudaStream_t)stream>>>(
      xs, ldx, rows, B, T, C, mean, var, eps, w, dpool, lddp, scalar, g, ldg, dw, dbeta);
  return post_launch("pool_bn_eval_bwd_kernel");
}

int fvit_stem_conv_dgrad(const void* dz16, int64_t lddz, int32_t B, int32_t H, int32_t W, const float* wgt,
                         int32_t cout, const float* scalar, float* dx, void* stream) {
  FVIT_CHECK(dz16 && wgt && scalar && dx && B > 0 && H > 0 && W > 0 && cout > 0 && cout <= 512 && lddz >= cout,
             "fvit_stem_conv_dgrad: bad arguments");
  const int H1 = (H + 1) / 2, W1 = (W + 1) / 2;
  FVIT_CHECK(B <= 65535 && (H1 + SD_OWN - 1) / SD_OWN <= 65535, "fvit_stem_conv_dgrad: B=%d H=%d too large", B, H);
  const int vec = lddz % 8 == 0 && reinterpret_cast<uintptr_t>(dz16) % 16 == 0;
  const size_t smem = ((size_t)cout * 28 + (size_t)SD_WIN * SD_WIN * 27) * sizeof(float);
  if (smem > 48 * 1024)
    FVIT_CUDA(cudaFuncSetAttribute(stem_conv_dgrad_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  dim3 grid((unsigned)((W1 + SD_OWN - 1) / SD_OWN), (unsigned)((H1 + SD_OWN - 1) / SD_OWN), (unsigned)B);
  stem_conv_dgrad_kernel<<<grid, 256, smem, (cudaStream_t)stream>>>((const __half*)dz16, lddz, vec, H, W, H1, W1, wgt,
                                                                     cout, scalar, dx);
  return post_launch("stem_conv_dgrad_kernel");
}

int fvit_stem_col2im(const float* dcol, int64_t ldc, int32_t B, int32_t cin, int32_t H, int32_t W, float* dx,
                     void* stream) {
  FVIT_CHECK(dcol && dx && B > 0 && H > 0 && W > 0 && ldc >= 9 * (int64_t)cin, "fvit_stem_col2im: bad arguments");
  FVIT_CHECK(cin >= 1 && cin <= FVIT_STEM_MAX_CIN, "fvit_stem_col2im: in_chans=%d must be in [1, %d]", cin,
             FVIT_STEM_MAX_CIN);
  const int H1 = (H + 1) / 2, W1 = (W + 1) / 2;
  FVIT_CHECK(B <= 65535 && (H1 + SD_OWN - 1) / SD_OWN <= 65535, "fvit_stem_col2im: B=%d H=%d too large", B, H);
  dim3 grid((unsigned)((W1 + SD_OWN - 1) / SD_OWN), (unsigned)((H1 + SD_OWN - 1) / SD_OWN), (unsigned)B);
  stem_col2im_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(dcol, ldc, cin, H, W, H1, W1, dx);
  return post_launch("stem_col2im_kernel");
}

}  // extern "C"
