// Multi-scale deformable attention core (MSDeformAttn of the DINO and MOTRv2 transformers): the bilinear gather of
// value rows at fractional per-level sampling locations, weighted and summed per query-head, and its backward.
// Semantics are grid_sample(mode='bilinear', padding_mode='zeros', align_corners=False) per level. Contracts are in
// include/fvit.h ("Multi-scale deformable attention").
//
// Layout of the work: one group of G lanes (G a power of two <= 32) serves one (n, q, m). Each lane owns VEC
// consecutive channels (float4 reads of the corner rows when D % 4 == 0 and the pointers are 16-byte aligned,
// scalar otherwise) and loops over ceil(D / (VEC * G)) channel chunks, so any D works. The group's sampling locations
// and weights are loaded once, one sample per lane, and handed around by shuffles. Level shapes and start rows sit in
// shared memory. Lanes past the last group mirror it, so that every shuffle runs with the full warp.
#include "../../include/fvit.h"
#include "common.h"

namespace fvit {
namespace {

constexpr int kMsdaThreads = 256;
constexpr unsigned kFull = 0xffffffffu;

template <int VEC>
struct Chunk {
  float v[VEC];
};

template <int VEC>
__device__ __forceinline__ Chunk<VEC> zero_chunk() {
  Chunk<VEC> r;
#pragma unroll
  for (int i = 0; i < VEC; ++i) r.v[i] = 0.f;
  return r;
}

template <int VEC>
__device__ __forceinline__ Chunk<VEC> load_chunk(const float* __restrict__ p) {
  Chunk<VEC> r;
  if constexpr (VEC == 4) {
    const float4 t = __ldg(reinterpret_cast<const float4*>(p));
    r.v[0] = t.x, r.v[1] = t.y, r.v[2] = t.z, r.v[3] = t.w;
  } else {
    r.v[0] = __ldg(p);
  }
  return r;
}

template <int VEC>
__device__ __forceinline__ void store_chunk(float* p, const Chunk<VEC>& c) {
  if constexpr (VEC == 4)
    *reinterpret_cast<float4*>(p) = make_float4(c.v[0], c.v[1], c.v[2], c.v[3]);
  else
    *p = c.v[0];
}

// p[0 .. VEC) += s * c: one red.global.add.v4.f32 on sm_90 for VEC 4 (that instruction flushes denormals to zero)
template <int VEC>
__device__ __forceinline__ void red_add(float* p, float s, const Chunk<VEC>& c) {
  if constexpr (VEC == 4)
    atomicAdd(reinterpret_cast<float4*>(p), make_float4(s * c.v[0], s * c.v[1], s * c.v[2], s * c.v[3]));
  else
    atomicAdd(p, s * c.v[0]);
}

// Level geometry into shared memory. A level whose rows do not lie inside [0, S) gets H = W = 0 and reads nothing, so
// spatial_shapes / level_start_index that disagree with value never address memory outside it.
__device__ __forceinline__ void load_levels(const int64_t* __restrict__ shapes, const int64_t* __restrict__ starts,
                                            int L, int S, int* s_h, int* s_w, int* s_start) {
  if (threadIdx.x < L) {
    const long long h = shapes[2 * threadIdx.x], w = shapes[2 * threadIdx.x + 1], st = starts[threadIdx.x];
    const bool ok = h >= 0 && w >= 0 && st >= 0 && h <= S && w <= S && st + h * w <= S;
    s_h[threadIdx.x] = ok ? (int)h : 0;
    s_w[threadIdx.x] = ok ? (int)w : 0;
    s_start[threadIdx.x] = ok ? (int)st : 0;
  }
  __syncthreads();
}

struct Bilinear {
  bool in;                // the sample contributes at all: h > -1, w > -1, h < H, w < W
  bool c1, c2, c3, c4;    // corners (h0, w0), (h0, w0 + 1), (h0 + 1, w0), (h0 + 1, w0 + 1) lie inside the map
  float lh, lw, hh, hw;   // fractional parts of h and w, and their complements
  long long row;          // pixel row of corner 1 (read only through c1..c4)
};

// sampling location (x, y) in [0, 1] of a level with H x W pixels; pixel centres at h = y*H - 0.5, w = x*W - 0.5
__device__ __forceinline__ Bilinear bilinear(float x, float y, int H, int W, int start) {
  Bilinear b;
  const float h = y * (float)H - 0.5f, w = x * (float)W - 0.5f;
  b.in = h > -1.f && w > -1.f && h < (float)H && w < (float)W;
  const float hf = floorf(h), wf = floorf(w);
  const int h0 = b.in ? (int)hf : -2, w0 = b.in ? (int)wf : -2;
  b.lh = h - hf, b.lw = w - wf, b.hh = 1.f - b.lh, b.hw = 1.f - b.lw;
  const bool top = h0 >= 0, bot = h0 + 1 < H, lef = w0 >= 0, rig = w0 + 1 < W;
  b.c1 = b.in && top && lef, b.c2 = b.in && top && rig, b.c3 = b.in && bot && lef, b.c4 = b.in && bot && rig;
  b.row = (long long)start + (long long)h0 * W + w0;
  return b;
}

struct MsdaGeom {
  long long groups;  // N * Lq * M
  int S, Lq, M, D, L, P, G;
};

// out[n, q, m*D + c] = sum_{l, p} attn[n, q, m, l, p] * bilinear(value[n, level l, m, c], loc[n, q, m, l, p])
template <int VEC>
__global__ void __launch_bounds__(kMsdaThreads)
    msda_fwd_kernel(const float* __restrict__ value, const int64_t* __restrict__ shapes,
                    const int64_t* __restrict__ starts, const float* __restrict__ loc, const float* __restrict__ attn,
                    float* __restrict__ out, MsdaGeom q) {
  __shared__ int s_h[FVIT_MSDA_MAX_LEVELS], s_w[FVIT_MSDA_MAX_LEVELS], s_start[FVIT_MSDA_MAX_LEVELS];
  load_levels(shapes, starts, q.L, q.S, s_h, s_w, s_start);
  const int G = q.G, gl = threadIdx.x & (G - 1);
  const long long grp = (blockIdx.x * (long long)blockDim.x + threadIdx.x) / G;
  const bool live = grp < q.groups;
  const long long g = live ? grp : q.groups - 1;
  const long long n = g / ((long long)q.Lq * q.M);
  const int m = (int)(g % q.M);
  const long long LP = (long long)q.L * q.P;
  const long long vstride = (long long)q.M * q.D;  // elements between consecutive pixels of value
  const float* __restrict__ vbase = value + n * q.S * vstride + (long long)m * q.D;
  const float* __restrict__ lbase = loc + g * LP * 2;
  const float* __restrict__ abase = attn + g * LP;
  const int nvec = q.D / VEC;
  for (int c0 = 0; c0 < nvec; c0 += G) {
    const int cv = c0 + gl;
    const bool cok = live && cv < nvec;
    const float* __restrict__ vc = vbase + (long long)cv * VEC;
    Chunk<VEC> acc = zero_chunk<VEC>();
    for (long long s0 = 0; s0 < LP; s0 += G) {
      float x = 0.f, y = 0.f, a = 0.f;
      if (s0 + gl < LP) {
        x = __ldg(lbase + 2 * (s0 + gl));
        y = __ldg(lbase + 2 * (s0 + gl) + 1);
        a = __ldg(abase + s0 + gl);
      }
      const int ns = (int)min((long long)G, LP - s0);
      for (int j = 0; j < ns; ++j) {
        const float sx = __shfl_sync(kFull, x, j, G), sy = __shfl_sync(kFull, y, j, G);
        const float sa = __shfl_sync(kFull, a, j, G);
        const int l = (int)((s0 + j) / q.P);
        const int W = s_w[l];
        const Bilinear b = bilinear(sx, sy, s_h[l], W, s_start[l]);
        if (!b.in || !cok) continue;
        const float w1 = b.hh * b.hw, w2 = b.hh * b.lw, w3 = b.lh * b.hw, w4 = b.lh * b.lw;
        const Chunk<VEC> v1 = b.c1 ? load_chunk<VEC>(vc + b.row * vstride) : zero_chunk<VEC>();
        const Chunk<VEC> v2 = b.c2 ? load_chunk<VEC>(vc + (b.row + 1) * vstride) : zero_chunk<VEC>();
        const Chunk<VEC> v3 = b.c3 ? load_chunk<VEC>(vc + (b.row + W) * vstride) : zero_chunk<VEC>();
        const Chunk<VEC> v4 = b.c4 ? load_chunk<VEC>(vc + (b.row + W + 1) * vstride) : zero_chunk<VEC>();
#pragma unroll
        for (int i = 0; i < VEC; ++i) {
          const float val = w1 * v1.v[i] + w2 * v2.v[i] + w3 * v3.v[i] + w4 * v4.v[i];
          acc.v[i] = fmaf(sa, val, acc.v[i]);
        }
      }
    }
    if (cok) store_chunk<VEC>(out + g * q.D + (long long)cv * VEC, acc);
  }
}

// Where the backward puts a corner's s * grad_out * attn into grad_value. FloatSink: fp32 vector atomics, whose order
// of additions is not deterministic. FixedSink: int64 fixed point in units of 2^-k, one round-to-nearest per
// contribution (the fp32 product of the float path, scaled by 2^k exactly); integer addition is associative, so the
// sums do not depend on the order of the samples.
struct FloatSink {
  float* base;
  template <int VEC>
  __device__ __forceinline__ void add(float* p, float s, const Chunk<VEC>& c) const {
    red_add<VEC>(p, s, c);
  }
};

struct FixedSink {
  unsigned long long* base;
  double scale;  // 2^k
  template <int VEC>
  __device__ __forceinline__ void add(unsigned long long* p, float s, const Chunk<VEC>& c) const {
#pragma unroll
    for (int i = 0; i < VEC; ++i) atomicAdd(p + i, (unsigned long long)__double2ll_rn((double)(s * c.v[i]) * scale));
  }
};

// Backward: grad_value gets every sample's corner weight * attn * grad_out through the sink; grad_attn and grad_loc of
// each sample are reduced over the group's channels by shuffles and written by lane 0 of the group, so they need no
// atomics and are deterministic. Every element of grad_loc and grad_attn is written.
template <int VEC, class Sink>
__device__ __forceinline__ void msda_bwd_body(const float* __restrict__ value, const int* s_h, const int* s_w,
                                              const int* s_start, const float* __restrict__ loc,
                                              const float* __restrict__ attn, const float* __restrict__ grad_out,
                                              const Sink& sink, float* __restrict__ grad_loc,
                                              float* __restrict__ grad_attn, const MsdaGeom& q) {
  const int G = q.G, gl = threadIdx.x & (G - 1);
  const long long grp = (blockIdx.x * (long long)blockDim.x + threadIdx.x) / G;
  const bool live = grp < q.groups;
  const long long g = live ? grp : q.groups - 1;
  const long long n = g / ((long long)q.Lq * q.M);
  const int m = (int)(g % q.M);
  const long long LP = (long long)q.L * q.P;
  const long long vstride = (long long)q.M * q.D;
  const long long vofs = n * q.S * vstride + (long long)m * q.D;
  const float* __restrict__ lbase = loc + g * LP * 2;
  const float* __restrict__ abase = attn + g * LP;
  const float* __restrict__ gobase = grad_out + g * q.D;
  const int nvec = q.D / VEC;
  // the first channel chunk's grad_out stays in registers (the only chunk for D <= VEC * G, e.g. DINO's D = 32)
  const Chunk<VEC> go0 = (live && gl < nvec) ? load_chunk<VEC>(gobase + gl * VEC) : zero_chunk<VEC>();
  for (long long s0 = 0; s0 < LP; s0 += G) {
    float x = 0.f, y = 0.f, a = 0.f;
    if (s0 + gl < LP) {
      x = __ldg(lbase + 2 * (s0 + gl));
      y = __ldg(lbase + 2 * (s0 + gl) + 1);
      a = __ldg(abase + s0 + gl);
    }
    const int ns = (int)min((long long)G, LP - s0);
    for (int j = 0; j < ns; ++j) {
      const float sx = __shfl_sync(kFull, x, j, G), sy = __shfl_sync(kFull, y, j, G);
      const float sa = __shfl_sync(kFull, a, j, G);
      const int l = (int)((s0 + j) / q.P);
      const int H = s_h[l], W = s_w[l];
      const Bilinear b = bilinear(sx, sy, H, W, s_start[l]);
      float ga = 0.f, gh = 0.f, gw = 0.f;  // d/d attn, d/dh and d/dw, this lane's channels
      if (b.in && live) {
        const float w1 = b.hh * b.hw, w2 = b.hh * b.lw, w3 = b.lh * b.hw, w4 = b.lh * b.lw;
        for (int c0 = 0; c0 < nvec; c0 += G) {
          const int cv = c0 + gl;
          if (cv >= nvec) break;
          const long long c = (long long)cv * VEC;
          const Chunk<VEC> go = c0 == 0 ? go0 : load_chunk<VEC>(gobase + c);
          const float* __restrict__ vc = value + vofs + c;
          auto* gv = sink.base + vofs + c;
          const Chunk<VEC> v1 = b.c1 ? load_chunk<VEC>(vc + b.row * vstride) : zero_chunk<VEC>();
          const Chunk<VEC> v2 = b.c2 ? load_chunk<VEC>(vc + (b.row + 1) * vstride) : zero_chunk<VEC>();
          const Chunk<VEC> v3 = b.c3 ? load_chunk<VEC>(vc + (b.row + W) * vstride) : zero_chunk<VEC>();
          const Chunk<VEC> v4 = b.c4 ? load_chunk<VEC>(vc + (b.row + W + 1) * vstride) : zero_chunk<VEC>();
          Chunk<VEC> tg;  // grad_out * attention weight
#pragma unroll
          for (int i = 0; i < VEC; ++i) {
            tg.v[i] = sa * go.v[i];
            const float val = w1 * v1.v[i] + w2 * v2.v[i] + w3 * v3.v[i] + w4 * v4.v[i];
            ga = fmaf(go.v[i], val, ga);
            const float dh = b.hw * (v3.v[i] - v1.v[i]) + b.lw * (v4.v[i] - v2.v[i]);
            const float dw = b.hh * (v2.v[i] - v1.v[i]) + b.lh * (v4.v[i] - v3.v[i]);
            gh = fmaf(tg.v[i], dh, gh);
            gw = fmaf(tg.v[i], dw, gw);
          }
          if (b.c1) sink.template add<VEC>(gv + b.row * vstride, w1, tg);
          if (b.c2) sink.template add<VEC>(gv + (b.row + 1) * vstride, w2, tg);
          if (b.c3) sink.template add<VEC>(gv + (b.row + W) * vstride, w3, tg);
          if (b.c4) sink.template add<VEC>(gv + (b.row + W + 1) * vstride, w4, tg);
        }
      }
      for (int o = G >> 1; o > 0; o >>= 1) {
        ga += __shfl_xor_sync(kFull, ga, o, G);
        gh += __shfl_xor_sync(kFull, gh, o, G);
        gw += __shfl_xor_sync(kFull, gw, o, G);
      }
      if (live && gl == 0) {
        const long long s = g * LP + s0 + j;
        grad_attn[s] = ga;
        grad_loc[2 * s] = gw * (float)W;
        grad_loc[2 * s + 1] = gh * (float)H;
      }
    }
  }
}

template <int VEC>
__global__ void __launch_bounds__(kMsdaThreads)
    msda_bwd_kernel(const float* __restrict__ value, const int64_t* __restrict__ shapes,
                    const int64_t* __restrict__ starts, const float* __restrict__ loc, const float* __restrict__ attn,
                    const float* __restrict__ grad_out, float* __restrict__ grad_value, float* __restrict__ grad_loc,
                    float* __restrict__ grad_attn, MsdaGeom q) {
  __shared__ int s_h[FVIT_MSDA_MAX_LEVELS], s_w[FVIT_MSDA_MAX_LEVELS], s_start[FVIT_MSDA_MAX_LEVELS];
  load_levels(shapes, starts, q.L, q.S, s_h, s_w, s_start);
  msda_bwd_body<VEC>(value, s_h, s_w, s_start, loc, attn, grad_out, FloatSink{grad_value}, grad_loc, grad_attn, q);
}

// ---- deterministic backward: bound pass, fixed-point accumulation, conversion ----

// bound[0] |= max |attn|, bound[1] |= max |grad_out|, as the bit patterns of non-negative floats, which order like
// their values; a NaN (sign cleared) sorts above inf, so a non-finite input leaves a pattern >= 0x7f800000. Maxima do
// not depend on the order. bound is zeroed before the launch.
__global__ void __launch_bounds__(kMsdaThreads)
    msda_bound_kernel(const float* __restrict__ attn, long long na, const float* __restrict__ grad_out, long long ng,
                      unsigned* __restrict__ bound) {
  const long long stride = (long long)gridDim.x * blockDim.x, i0 = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  unsigned ma = 0, mg = 0;
#pragma unroll 4
  for (long long i = i0; i < ng; i += stride) mg = max(mg, __float_as_uint(fabsf(__ldg(grad_out + i))));
  for (long long i = i0; i < na; i += stride) ma = max(ma, __float_as_uint(fabsf(__ldg(attn + i))));
  ma = __reduce_max_sync(kFull, ma);
  mg = __reduce_max_sync(kFull, mg);
  if ((threadIdx.x & 31) == 0) {
    atomicMax(bound, ma);
    atomicMax(bound + 1, mg);
  }
}

// Fixed-point exponent k of grad_value's sums (they count units of 2^-k); false if A = max |attn| or
// G = max |grad_out| is not finite.
//
// Bound: an element (n, pixel, m, c) of grad_value receives at most one contribution per sample of its (n, m), since
// a sample's four corners are distinct pixels; rows of different levels may coincide (level_start_index is not
// checked), so that is up to ns = Lq * L * P contributions. Each is w * (a * g) in fp32 with a corner weight w <= 1,
// |a| <= A, |g| <= G, so every partial or whole sum is at most B = ns * A * G (times (1 + 2^-24)^2 for the two fp32
// roundings). With B < 2^e <= 2B, k = 62 - e puts B * 2^k below 2^62; rounding adds at most ns / 2 < 2^62 units
// (ns < 2^35 for any attention_weights that fits in memory), so the sums stay below 2^63 in magnitude.
// Error: one contribution rounds by at most 2^-(k+1) <= B * 2^-62, so an element with ne contributions is within
// ne * B * 2^-62 <= ns^2 * A * G * 2^-62 of the exact sum of the fp32 contributions, before its conversion to fp32.
// At DINO's 5-scale encoder (ns = 1.8 M) that is 7e-7 * A * G.
__device__ __forceinline__ bool fixed_exponent(const unsigned* __restrict__ bound, long long ns, int* k) {
  const unsigned ab = bound[0], gb = bound[1];
  *k = 0;
  if (ab >= 0x7f800000u || gb >= 0x7f800000u) return false;
  const double B = (double)ns * (double)__uint_as_float(ab) * (double)__uint_as_float(gb);
  if (B > 0.0) {
    int e;
    frexp(B, &e);  // B = f * 2^e, f in [0.5, 1)
    *k = 62 - e;
  }
  return true;
}

// msda_bwd_kernel<1> with grad_value summed in int64 fixed point (acc, zeroed before the launch). One channel per
// lane, so each 64-bit atomic instruction of a group covers consecutive addresses; with msda_bwd_kernel<4>'s float4
// layout (four channels per lane) an instruction's addresses lie 32 bytes apart, and that variant took 2.2 to 2.4
// times as long at the README's four workloads on an H100.
__global__ void __launch_bounds__(kMsdaThreads)
    msda_bwd_fixed_kernel(const float* __restrict__ value, const int64_t* __restrict__ shapes,
                          const int64_t* __restrict__ starts, const float* __restrict__ loc,
                          const float* __restrict__ attn, const float* __restrict__ grad_out,
                          unsigned long long* __restrict__ acc, const unsigned* __restrict__ bound,
                          float* __restrict__ grad_loc, float* __restrict__ grad_attn, MsdaGeom q) {
  __shared__ int s_h[FVIT_MSDA_MAX_LEVELS], s_w[FVIT_MSDA_MAX_LEVELS], s_start[FVIT_MSDA_MAX_LEVELS];
  load_levels(shapes, starts, q.L, q.S, s_h, s_w, s_start);
  int k;
  // with a non-finite bound the sums are meaningless (and harmless: unsigned adds wrap); msda_fixed_to_float_kernel
  // writes NaN instead
  fixed_exponent(bound, (long long)q.Lq * q.L * q.P, &k);
  msda_bwd_body<1>(value, s_h, s_w, s_start, loc, attn, grad_out, FixedSink{acc, ldexp(1.0, k)}, grad_loc, grad_attn,
                   q);
}

// grad_value = acc * 2^-k (one rounding to double when |acc| > 2^53, exact scaling, one rounding to fp32), or NaN
// everywhere when the bound is not finite
__global__ void __launch_bounds__(kMsdaThreads)
    msda_fixed_to_float_kernel(const unsigned long long* __restrict__ acc, long long count,
                               const unsigned* __restrict__ bound, long long ns, float* __restrict__ grad_value) {
  int k;
  const bool finite = fixed_exponent(bound, ns, &k);
  const double unit = ldexp(1.0, -k);
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < count; i += stride)
    grad_value[i] = finite ? (float)((double)(long long)acc[i] * unit) : __int_as_float(0x7fc00000);
}

// lanes per group: the channel vectors of one head rounded up to a power of two, at most a warp
int group_lanes(int nvec) {
  int g = 1;
  while (g < nvec && g < 32) g <<= 1;
  return g;
}

bool aligned16(const void* p) { return ((uintptr_t)p & 15u) == 0; }

// blocks of a grid-stride pass over count elements: enough to fill an H100 (132 SMs x 8 blocks), at least one
unsigned stream_blocks(long long count) {
  const long long b = ceil_div64(count, kMsdaThreads);
  return b < 1 ? 1u : b > 1056 ? 1056u : (unsigned)b;
}

int check_geom(const char* fn, int32_t N, int32_t S, int32_t M, int32_t D, int32_t Lq, int32_t L, int32_t P,
               MsdaGeom* q) {
  FVIT_CHECK(L <= FVIT_MSDA_MAX_LEVELS, "%s: %d feature levels; at most %d (FVIT_MSDA_MAX_LEVELS) are supported", fn,
             L, FVIT_MSDA_MAX_LEVELS);
  FVIT_CHECK(N >= 0 && S >= 0 && M >= 0 && Lq >= 0 && D >= 1 && L >= 1 && P >= 1,
             "%s: bad sizes N=%d S=%d M=%d D=%d Lq=%d L=%d P=%d", fn, N, S, M, D, Lq, L, P);
  q->groups = (long long)N * Lq * M;
  q->S = S, q->Lq = Lq, q->M = M, q->D = D, q->L = L, q->P = P;
  return 0;
}

}  // namespace
}  // namespace fvit

using namespace fvit;

int fvit_msda_fwd(const float* value, const int64_t* spatial_shapes, const int64_t* level_start_index,
                  const float* sampling_locations, const float* attention_weights, int32_t N, int32_t S, int32_t M,
                  int32_t D, int32_t Lq, int32_t L, int32_t P, float* out, void* stream) {
  MsdaGeom q;
  if (int rc = check_geom("fvit_msda_fwd", N, S, M, D, Lq, L, P, &q)) return rc;
  if (q.groups == 0) return 0;
  FVIT_CHECK(value && spatial_shapes && level_start_index && sampling_locations && attention_weights && out,
             "fvit_msda_fwd: null pointer");
  const bool vec = D % 4 == 0 && aligned16(value) && aligned16(out);
  q.G = group_lanes(vec ? D / 4 : D);
  const long long blocks = ceil_div64(q.groups * q.G, kMsdaThreads);
  FVIT_CHECK(blocks <= 0x7fffffffLL, "fvit_msda_fwd: %lld query-heads is too many for one launch", q.groups);
  if (vec) {
    msda_fwd_kernel<4><<<(unsigned)blocks, kMsdaThreads, 0, (cudaStream_t)stream>>>(
        value, spatial_shapes, level_start_index, sampling_locations, attention_weights, out, q);
    return post_launch("msda_fwd_kernel<4>");
  }
  msda_fwd_kernel<1><<<(unsigned)blocks, kMsdaThreads, 0, (cudaStream_t)stream>>>(
      value, spatial_shapes, level_start_index, sampling_locations, attention_weights, out, q);
  return post_launch("msda_fwd_kernel<1>");
}

int fvit_msda_bwd(const float* value, const int64_t* spatial_shapes, const int64_t* level_start_index,
                  const float* sampling_locations, const float* attention_weights, const float* grad_out, int32_t N,
                  int32_t S, int32_t M, int32_t D, int32_t Lq, int32_t L, int32_t P, float* grad_value,
                  float* grad_sampling_locations, float* grad_attention_weights, void* stream) {
  MsdaGeom q;
  if (int rc = check_geom("fvit_msda_bwd", N, S, M, D, Lq, L, P, &q)) return rc;
  if (q.groups == 0) return 0;
  FVIT_CHECK(value && spatial_shapes && level_start_index && sampling_locations && attention_weights && grad_out &&
                 grad_value && grad_sampling_locations && grad_attention_weights,
             "fvit_msda_bwd: null pointer");
  const bool vec = D % 4 == 0 && aligned16(value) && aligned16(grad_out) && aligned16(grad_value);
  q.G = group_lanes(vec ? D / 4 : D);
  const long long blocks = ceil_div64(q.groups * q.G, kMsdaThreads);
  FVIT_CHECK(blocks <= 0x7fffffffLL, "fvit_msda_bwd: %lld query-heads is too many for one launch", q.groups);
  if (vec) {
    msda_bwd_kernel<4><<<(unsigned)blocks, kMsdaThreads, 0, (cudaStream_t)stream>>>(
        value, spatial_shapes, level_start_index, sampling_locations, attention_weights, grad_out, grad_value,
        grad_sampling_locations, grad_attention_weights, q);
    return post_launch("msda_bwd_kernel<4>");
  }
  msda_bwd_kernel<1><<<(unsigned)blocks, kMsdaThreads, 0, (cudaStream_t)stream>>>(
      value, spatial_shapes, level_start_index, sampling_locations, attention_weights, grad_out, grad_value,
      grad_sampling_locations, grad_attention_weights, q);
  return post_launch("msda_bwd_kernel<1>");
}

int fvit_msda_bwd_deterministic(const float* value, const int64_t* spatial_shapes, const int64_t* level_start_index,
                                const float* sampling_locations, const float* attention_weights, const float* grad_out,
                                int32_t N, int32_t S, int32_t M, int32_t D, int32_t Lq, int32_t L, int32_t P,
                                float* grad_value, float* grad_sampling_locations, float* grad_attention_weights,
                                int64_t* scratch, float* workspace, void* stream) {
  MsdaGeom q;
  if (int rc = check_geom("fvit_msda_bwd_deterministic", N, S, M, D, Lq, L, P, &q)) return rc;
  const long long nvalue = (long long)N * S * M * D, ns = (long long)Lq * L * P;
  if (q.groups == 0 && nvalue == 0) return 0;
  FVIT_CHECK(value && spatial_shapes && level_start_index && sampling_locations && attention_weights && grad_out &&
                 grad_value && grad_sampling_locations && grad_attention_weights && scratch && workspace,
             "fvit_msda_bwd_deterministic: null pointer");
  q.G = group_lanes(D);  // one channel per lane for any D and alignment (msda_bwd_fixed_kernel)
  const long long blocks = ceil_div64(q.groups * q.G, kMsdaThreads);
  FVIT_CHECK(blocks <= 0x7fffffffLL, "fvit_msda_bwd_deterministic: %lld query-heads is too many for one launch",
             q.groups);
  cudaStream_t st = (cudaStream_t)stream;
  unsigned* bound = reinterpret_cast<unsigned*>(workspace);
  unsigned long long* acc = reinterpret_cast<unsigned long long*>(scratch);
  FVIT_CUDA(cudaMemsetAsync(bound, 0, FVIT_MSDA_DET_WORKSPACE * sizeof(float), st));
  FVIT_CUDA(cudaMemsetAsync(acc, 0, (size_t)nvalue * sizeof(int64_t), st));
  const long long na = q.groups * L * P, ng = q.groups * D;
  msda_bound_kernel<<<stream_blocks(std::max(na, ng)), kMsdaThreads, 0, st>>>(attention_weights, na, grad_out, ng,
                                                                               bound);
  if (int rc = post_launch("msda_bound_kernel")) return rc;
  if (q.groups > 0) {
    msda_bwd_fixed_kernel<<<(unsigned)blocks, kMsdaThreads, 0, st>>>(
        value, spatial_shapes, level_start_index, sampling_locations, attention_weights, grad_out, acc, bound,
        grad_sampling_locations, grad_attention_weights, q);
    if (int rc = post_launch("msda_bwd_fixed_kernel")) return rc;
  }
  if (nvalue == 0) return 0;
  msda_fixed_to_float_kernel<<<stream_blocks(nvalue), kMsdaThreads, 0, st>>>(acc, nvalue, bound, ns, grad_value);
  return post_launch("msda_fixed_to_float_kernel");
}
