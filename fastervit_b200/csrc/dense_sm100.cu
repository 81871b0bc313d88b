// Backward of the dense-prediction outputs (forward_levels / forward_features / the backbone's norm{i} in train mode):
// the NCHW fp32 map gradient dy of out[b][c][t] = BN(xs[row_map[b*T+t]][c]) back into the level's token-major fp32
// gradient rows, with the batch-statistics BatchNorm folded in. Two passes, both over 32 x 32 (token, channel) tiles
// transposed through shared memory so that the NCHW planes (contiguous in t) and the token rows (contiguous in c) are
// read and written coalesced:
//   stats : s1[c] = sum dy, s2[c] = sum dy * xhat, amax = max |dy|   (all requested outputs, before the gradient
//           scale S is known: S = 2^floor(log2(64 / amax)) over every output, fvit_grad_scale_finalize)
//   apply : g[row][c] += S * w * rstd * (dy - s1/N - xhat * s2/N)  (N = B*T), dw += s2, dbeta += s1
// Without a BatchNorm (raw forward_levels maps) the stats pass only takes amax and apply is g += S * dy.
// Contracts are in include/fvit.h.
#include "../../include/fvit.h"
#include "common.h"

namespace fvit {

// one block = (32, 8) threads, 32 channels [c0, c0+32) of a grid-strided list of (image, 32-token tile) items.
// Thread (x, y) accumulates channels c0 + y + 8k (k < 4) over tokens t0 + x; lanes are reduced at the end.
__global__ void __launch_bounds__(256)
feature_map_bwd_stats_kernel(const float* __restrict__ dy, const float* __restrict__ xs, long long ldx,
                             const int* __restrict__ row_map, int B, int T, int C, const float* __restrict__ mean,
                             const float* __restrict__ rstd, float* __restrict__ s1, float* __restrict__ s2,
                             float* __restrict__ amax) {
  __shared__ float xh[32][33];
  const int c0 = blockIdx.y * 32;
  const int ntt = (T + 31) / 32;
  const bool bn = mean != nullptr;
  float a1[4] = {0.f, 0.f, 0.f, 0.f}, a2[4] = {0.f, 0.f, 0.f, 0.f}, mx = 0.f;
  for (long long item = blockIdx.x; item < (long long)B * ntt; item += gridDim.x) {
    const int b = (int)(item / ntt), t0 = (int)(item % ntt) * 32;
    const int t = t0 + threadIdx.x;
    // the dy loads are issued before the xs tile is staged, so both streams are in flight together
    float d[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const int c = c0 + threadIdx.y + 8 * k;
      d[k] = (t < T && c < C) ? dy[((long long)b * C + c) * T + t] : 0.f;
    }
    if (bn) {
      __syncthreads();   // previous item's reads of xh are done
      const int c = c0 + threadIdx.x;
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const int i = threadIdx.y + 8 * k, tt = t0 + i;
        float v = 0.f;
        if (tt < T && c < C) {
          const long long row = row_map ? row_map[(long long)b * T + tt] : (long long)b * T + tt;
          v = (xs[row * ldx + c] - __ldg(mean + c)) * __ldg(rstd + c);
        }
        xh[i][threadIdx.x] = v;
      }
      __syncthreads();
    }
#pragma unroll
    for (int k = 0; k < 4; ++k) {   // (out-of-range entries are zeros: they add nothing)
      mx = fmaxf(mx, fabsf(d[k]));
      if (bn) {
        a1[k] += d[k];
        a2[k] = fmaf(d[k], xh[threadIdx.x][threadIdx.y + 8 * k], a2[k]);
      }
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  if (threadIdx.x == 0 && mx > 0.f) atomicMax(reinterpret_cast<int*>(amax), __float_as_int(mx));   // (|dy| >= 0: int order)
  if (!bn) return;
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    float u = a1[k], v = a2[k];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      u += __shfl_xor_sync(0xffffffffu, u, o);
      v += __shfl_xor_sync(0xffffffffu, v, o);
    }
    const int c = c0 + threadIdx.y + 8 * k;
    if (threadIdx.x == 0 && c < C) {
      atomicAdd(s1 + c, u);
      atomicAdd(s2 + c, v);
    }
  }
}

// grid = (token tiles, channel tiles, images); the dy tile is staged [c][t] (coalesced NCHW reads), then every thread
// owns one (token, channel) with the channel along the lane: coalesced xs reads and g read-modify-writes.
__global__ void __launch_bounds__(256)
feature_map_bwd_apply_kernel(const float* __restrict__ dy, const float* __restrict__ xs, long long ldx,
                             const int* __restrict__ row_map, int T, int C, const float* __restrict__ mean,
                             const float* __restrict__ rstd, const float* __restrict__ w, const float* __restrict__ s1,
                             const float* __restrict__ s2, float inv_n, const float* __restrict__ gs,
                             float* __restrict__ g, long long ldg) {
  __shared__ float tile[32][33];
  const int b = blockIdx.z, t0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
  for (int i = threadIdx.y; i < 32; i += 8) {
    const int c = c0 + i, t = t0 + threadIdx.x;
    tile[i][threadIdx.x] = (t < T && c < C) ? dy[((long long)b * C + c) * T + t] : 0.f;
  }
  __syncthreads();
  const int c = c0 + threadIdx.x;
  if (c >= C) return;
  const float S = __ldg(gs);
  float k1 = S, m1 = 0.f, m2 = 0.f, mu = 0.f, rs = 1.f;
  if (mean) {
    mu = __ldg(mean + c);
    rs = __ldg(rstd + c);
    k1 = S * __ldg(w + c) * rs;
    m1 = __ldg(s1 + c) * inv_n;
    m2 = __ldg(s2 + c) * inv_n;
  }
  for (int i = threadIdx.y; i < 32; i += 8) {
    const int t = t0 + i;
    if (t >= T) break;
    const long long row = row_map ? row_map[(long long)b * T + t] : (long long)b * T + t;
    const float d = tile[threadIdx.x][i];
    float dx = d;
    if (mean) {
      const float xhat = (xs[row * ldx + c] - mu) * rs;
      dx = d - m1 - xhat * m2;
    }
    g[row * ldg + c] += k1 * dx;
  }
}

// The same transposes for a running-statistics BatchNorm (eval mode): the map gradient is a per-channel scale of dy, so
// the apply reads dy and read-modify-writes g, and never touches xs (no mean(dy) / mean(dy*xhat) terms). With no xs
// stream to overlap, a block takes 32 channels x 64 tokens and every thread issues its 8 dy loads, then its 8 g loads,
// before any store: enough bytes in flight per SM for the HBM-bound pass.
constexpr int kEvalTok = 64;
__global__ void __launch_bounds__(256)
feature_map_eval_bwd_apply_kernel(const float* __restrict__ dy, const int* __restrict__ row_map, int T, int C,
                                  const float* __restrict__ rstd, const float* __restrict__ w,
                                  const float* __restrict__ gs, float* __restrict__ g, long long ldg) {
  __shared__ float tile[32][kEvalTok + 1];
  const int b = blockIdx.z, t0 = blockIdx.x * kEvalTok, c0 = blockIdx.y * 32;
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const int i = threadIdx.y + 8 * k, c = c0 + i;
#pragma unroll
    for (int h = 0; h < kEvalTok / 32; ++h) {
      const int t = t0 + 32 * h + threadIdx.x;
      tile[i][32 * h + threadIdx.x] = (t < T && c < C) ? dy[((long long)b * C + c) * T + t] : 0.f;
    }
  }
  __syncthreads();
  const int c = c0 + threadIdx.x;
  if (c >= C) return;
  float k1 = __ldg(gs);
  if (w) k1 = k1 * __ldg(w + c) * __ldg(rstd + c);
  constexpr int kPer = kEvalTok / 8;
  long long row[kPer];
  float gv[kPer];
#pragma unroll
  for (int k = 0; k < kPer; ++k) {
    const int t = t0 + threadIdx.y + 8 * k;
    row[k] = t < T ? (row_map ? (long long)row_map[(long long)b * T + t] : (long long)b * T + t) : -1;
  }
#pragma unroll
  for (int k = 0; k < kPer; ++k) gv[k] = row[k] >= 0 ? g[row[k] * ldg + c] : 0.f;
#pragma unroll
  for (int k = 0; k < kPer; ++k)
    if (row[k] >= 0) g[row[k] * ldg + c] = gv[k] + k1 * tile[threadIdx.x][threadIdx.y + 8 * k];
}

// dw[c] += s2[c] * scalar, dbeta[c] += s1[c] * scalar
__global__ void bn_affine_grad_kernel(const float* __restrict__ s1, const float* __restrict__ s2,
                                      const float* __restrict__ scalar, int C, float* __restrict__ dw,
                                      float* __restrict__ dbeta) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  const float sc = scalar ? __ldg(scalar) : 1.f;
  dw[c] += s2[c] * sc;
  dbeta[c] += s1[c] * sc;
}

// gs = {S, 1/S}, S = 2^floor(log2(target / amax)) clamped like grad_scale_init_kernel (train_sm100.cu)
__global__ void grad_scale_finalize_kernel(const float* __restrict__ amax, float target, float* __restrict__ gs) {
  const float m = *amax;
  float S = 1.f;
  if (m > 0.f && isfinite(m)) S = exp2f(floorf(log2f(target / m)));
  S = fminf(fmaxf(S, 1.f / 16777216.f), 16777216.f * 65536.f);
  gs[0] = S;
  gs[1] = 1.f / S;
}

// ---- backward of forward_head (avg-pool + Linear) in fp32
// pooled[r] = mean_t x[r][t] over rows r = b*C + c of an NCHW map: one warp per row, lanes along t
__global__ void nchw_row_mean_kernel(const float* __restrict__ x, long long rows, int T, float* __restrict__ pooled) {
  const long long r = (long long)blockIdx.x * (blockDim.x / 32) + threadIdx.x / 32;
  if (r >= rows) return;
  const int lane = threadIdx.x & 31;
  float s = 0.f;
  for (int t = lane; t < T; t += 32) s += x[r * T + t];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if (lane == 0) pooled[r] = s / (float)T;
}

// dfeats[b][c][t] = (sum_k dl[b][k] * W[k][c]) / T (W NULL: dl[b][c] / T). grid = (channel tiles of 128, B); the
// dlogits row is staged in shared memory in chunks, W is read along c (coalesced); the block's [128 x T] output slab
// is contiguous in NCHW and written linearly.
__global__ void __launch_bounds__(128)
head_eval_dgrad_kernel(const float* __restrict__ dl, long long ldl, int ncls, const float* __restrict__ W, int C, int T,
                       float* __restrict__ dfeats) {
  __shared__ float dls[128];
  __shared__ float dps[128];
  const int b = blockIdx.y, c0 = blockIdx.x * 128, c = c0 + threadIdx.x;
  float acc = 0.f;
  if (W) {
    for (int k0 = 0; k0 < ncls; k0 += 128) {
      __syncthreads();
      dls[threadIdx.x] = (k0 + threadIdx.x < ncls) ? dl[b * ldl + k0 + threadIdx.x] : 0.f;
      __syncthreads();
      if (c < C) {
        const int kn = min(128, ncls - k0);
        for (int j = 0; j < kn; ++j) acc = fmaf(dls[j], __ldg(W + (long long)(k0 + j) * C + c), acc);
      }
    }
  } else if (c < C) {
    acc = dl[b * ldl + c];
  }
  dps[threadIdx.x] = acc / (float)T;
  __syncthreads();
  const long long n = (long long)min(128, C - c0) * T;
  float* out = dfeats + ((long long)b * C + c0) * T;
  for (long long i = threadIdx.x; i < n; i += 128) out[i] = dps[i / T];
}

// dW[k][c] += sum_b dl[b][k] * pooled[b][c]; db[k] += sum_b dl[b][k]. grid = (channel tiles of 128, ncls): pooled is
// read along c (coalesced), the dlogits column value is the same for the whole block.
__global__ void __launch_bounds__(128)
head_eval_wgrad_kernel(const float* __restrict__ dl, long long ldl, int B, const float* __restrict__ pooled, int C,
                       float* __restrict__ dW, float* __restrict__ db) {
  const int k = blockIdx.y, c = blockIdx.x * 128 + threadIdx.x;
  if (c < C) {
    float acc = 0.f;
    for (int b = 0; b < B; ++b) acc = fmaf(__ldg(dl + b * ldl + k), __ldg(pooled + (long long)b * C + c), acc);
    dW[(long long)k * C + c] += acc;
  }
  if (db && blockIdx.x == 0 && threadIdx.x == 0) {
    float s = 0.f;
    for (int b = 0; b < B; ++b) s += dl[b * ldl + k];
    db[k] += s;
  }
}

}  // namespace fvit

using namespace fvit;

extern "C" {

int fvit_feature_map_bwd_stats(const float* dy, const float* xs, int64_t ldx, const int32_t* row_map, int32_t B,
                               int32_t T, int32_t C, const float* mean, const float* rstd, float* s1, float* s2,
                               float* amax, void* stream) {
  FVIT_CHECK(dy && amax && B > 0 && T > 0 && C > 0, "fvit_feature_map_bwd_stats: bad arguments");
  FVIT_CHECK(!mean || (xs && rstd && s1 && s2), "fvit_feature_map_bwd_stats: the BatchNorm mode needs xs, rstd, s1, s2");
  const long long items = (long long)B * ((T + 31) / 32);
  const int ctiles = (C + 31) / 32;
  // one wave of resident blocks (a second, partial wave would leave the grid-strided tail to a few blocks)
  static int per_sm = 0;
  if (per_sm == 0) {
    FVIT_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, feature_map_bwd_stats_kernel, 256, 0));
    if (per_sm < 1) per_sm = 1;
  }
  long long gx = (long long)num_sms() * per_sm / ctiles;
  if (gx < 1) gx = 1;
  if (gx > items) gx = items;
  feature_map_bwd_stats_kernel<<<dim3((unsigned)gx, (unsigned)ctiles), dim3(32, 8), 0, (cudaStream_t)stream>>>(
      dy, xs, ldx, row_map, B, T, C, mean, rstd, s1, s2, amax);
  return post_launch("feature_map_bwd_stats_kernel");
}

int fvit_feature_map_bwd(const float* dy, const float* xs, int64_t ldx, const int32_t* row_map, int32_t B, int32_t T,
                         int32_t C, const float* mean, const float* rstd, const float* w, const float* s1,
                         const float* s2, const float* gs, const float* scalar, float* g, int64_t ldg, float* dw,
                         float* dbeta, void* stream) {
  FVIT_CHECK(dy && gs && B > 0 && T > 0 && C > 0 && B <= 65535, "fvit_feature_map_bwd: bad arguments");
  FVIT_CHECK(!mean || (xs && rstd && w && s1 && s2), "fvit_feature_map_bwd: the BatchNorm mode needs xs, rstd, w, s1, s2");
  FVIT_CHECK((dw == nullptr) == (dbeta == nullptr) && (!dw || mean), "fvit_feature_map_bwd: dw / dbeta come in pairs "
             "and need the BatchNorm mode");
  if (g) {
    dim3 grid((T + 31) / 32, (C + 31) / 32, B);
    feature_map_bwd_apply_kernel<<<grid, dim3(32, 8), 0, (cudaStream_t)stream>>>(
        dy, xs, ldx, row_map, T, C, mean, rstd, w, s1, s2, 1.f / ((float)B * (float)T), gs, g, ldg);
    const int rc = post_launch("feature_map_bwd_apply_kernel");
    if (rc) return rc;
  }
  if (dw) {
    bn_affine_grad_kernel<<<ceil_div(C, 128), 128, 0, (cudaStream_t)stream>>>(s1, s2, scalar, C, dw, dbeta);
    return post_launch("bn_affine_grad_kernel");
  }
  return 0;
}

int fvit_feature_map_eval_bwd(const float* dy, const int32_t* row_map, int32_t B, int32_t T, int32_t C,
                              const float* rstd, const float* w, const float* s1, const float* s2, const float* gs,
                              const float* scalar, float* g, int64_t ldg, float* dw, float* dbeta, void* stream) {
  FVIT_CHECK(B > 0 && T > 0 && C > 0 && B <= 65535, "fvit_feature_map_eval_bwd: bad arguments");
  FVIT_CHECK((w == nullptr) == (rstd == nullptr), "fvit_feature_map_eval_bwd: w and rstd come in pairs");
  FVIT_CHECK(!g || (dy && gs), "fvit_feature_map_eval_bwd: the map gradient needs dy and gs");
  FVIT_CHECK((dw == nullptr) == (dbeta == nullptr) && (!dw || (w && s1 && s2)), "fvit_feature_map_eval_bwd: dw / dbeta "
             "come in pairs and need the BatchNorm mode (w, rstd) and s1, s2");
  if (g) {
    dim3 grid((T + kEvalTok - 1) / kEvalTok, (C + 31) / 32, B);
    feature_map_eval_bwd_apply_kernel<<<grid, dim3(32, 8), 0, (cudaStream_t)stream>>>(dy, row_map, T, C, rstd, w, gs,
                                                                                       g, ldg);
    const int rc = post_launch("feature_map_eval_bwd_apply_kernel");
    if (rc) return rc;
  }
  if (dw) {
    bn_affine_grad_kernel<<<ceil_div(C, 128), 128, 0, (cudaStream_t)stream>>>(s1, s2, scalar, C, dw, dbeta);
    return post_launch("bn_affine_grad_kernel");
  }
  return 0;
}

int fvit_head_eval_bwd(const float* dlogits, int64_t ldl, int32_t B, int32_t ncls, const float* feats, int32_t C,
                       int32_t T, const float* W, float* pooled_ws, float* dfeats, float* dW, float* db, void* stream) {
  FVIT_CHECK(dlogits && B > 0 && ncls > 0 && C > 0 && T > 0 && B <= 65535 && ncls <= 65535,
             "fvit_head_eval_bwd: bad arguments");
  FVIT_CHECK(W || ncls == C, "fvit_head_eval_bwd: an identity head (W NULL) has ncls == C");
  FVIT_CHECK(ldl >= ncls, "fvit_head_eval_bwd: ldl < ncls");
  FVIT_CHECK(!dW || (W && feats && (T == 1 || pooled_ws)), "fvit_head_eval_bwd: dW needs W, feats and (T > 1) pooled_ws");
  FVIT_CHECK(!db || W, "fvit_head_eval_bwd: db needs a Linear head");
  cudaStream_t st = (cudaStream_t)stream;
  if (dfeats) {
    head_eval_dgrad_kernel<<<dim3(ceil_div(C, 128), B), 128, 0, st>>>(dlogits, ldl, ncls, W, C, T, dfeats);
    const int rc = post_launch("head_eval_dgrad_kernel");
    if (rc) return rc;
  }
  if (dW) {
    const float* pooled = feats;
    if (T > 1) {
      const long long rows = (long long)B * C;
      nchw_row_mean_kernel<<<(unsigned)((rows + 7) / 8), 256, 0, st>>>(feats, rows, T, pooled_ws);
      const int rc = post_launch("nchw_row_mean_kernel");
      if (rc) return rc;
      pooled = pooled_ws;
    }
    head_eval_wgrad_kernel<<<dim3(ceil_div(C, 128), ncls), 128, 0, st>>>(dlogits, ldl, B, pooled, C, dW, db);
    return post_launch("head_eval_wgrad_kernel");
  }
  if (db) {   // (a bias without a weight gradient: the column sums alone, through the same kernel with no channels)
    head_eval_wgrad_kernel<<<dim3(1, ncls), 128, 0, st>>>(dlogits, ldl, B, nullptr, 0, nullptr, db);
    return post_launch("head_eval_wgrad_kernel");
  }
  return 0;
}

int fvit_grad_scale_finalize(const float* amax, float target, float* gs, void* stream) {
  FVIT_CHECK(amax && gs && target > 0, "fvit_grad_scale_finalize: bad arguments");
  grad_scale_finalize_kernel<<<1, 1, 0, (cudaStream_t)stream>>>(amax, target, gs);
  return post_launch("grad_scale_finalize_kernel");
}

}  // extern "C"
