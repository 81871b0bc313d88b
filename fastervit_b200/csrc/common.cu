// Library-level state of libfvit_sm100.so: error strings, launch counter, TMA descriptor encoding.
#include "common.h"

#include <cstring>
#include <mutex>
#include <unordered_map>

#include "../../include/fvit.h"

namespace fvit {

std::atomic<int64_t> g_launches{0};

char* err_buf() {
  static thread_local char buf[512] = {0};
  return buf;
}

int set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(err_buf(), 512, fmt, ap);
  va_end(ap);
  return 1;
}

static std::atomic<int> g_sm_limit{0};

int num_sms() {
  static int n = 0;
  if (n == 0) {
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) return 132;
    cudaDeviceProp p;
    if (cudaGetDeviceProperties(&p, dev) != cudaSuccess) return 132;
    n = p.multiProcessorCount;
  }
  const int lim = g_sm_limit.load(std::memory_order_relaxed);
  return (lim > 0 && lim < n) ? lim : n;
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*,
                                  const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                  const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode_fn() {
  static EncodeTiledFn fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) ==
            cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(p);
  });
  return fn;
}

static int encode_tmap_typed(CUtensorMap* out, const void* base, int rank, const uint64_t* dims,
                             const uint64_t* strides_bytes, const uint32_t* box, CUtensorMapSwizzle swz,
                             CUtensorMapDataType dtype);

int encode_tmap_16bit(CUtensorMap* out, const void* base, int rank, const uint64_t* dims,
                      const uint64_t* strides_bytes, const uint32_t* box, CUtensorMapSwizzle swz) {
  // FLOAT16 covers fp16 and bf16 alike for a tiled copy (no arithmetic on the elements).
  return encode_tmap_typed(out, base, rank, dims, strides_bytes, box, swz, CU_TENSOR_MAP_DATA_TYPE_FLOAT16);
}

static int encode_tmap_typed(CUtensorMap* out, const void* base, int rank, const uint64_t* dims,
                             const uint64_t* strides_bytes, const uint32_t* box, CUtensorMapSwizzle swz,
                             CUtensorMapDataType dtype) {
  EncodeTiledFn fn = get_encode_fn();
  if (!fn) return set_error("cuTensorMapEncodeTiled not available from the driver");
  if ((reinterpret_cast<uintptr_t>(base) & 15) != 0)
    return set_error("TMA base pointer %p is not 16-byte aligned", base);
  cuuint64_t gdim[5];
  cuuint64_t gstr[4];
  cuuint32_t bx[5];
  cuuint32_t es[5];
  for (int i = 0; i < rank; ++i) {
    gdim[i] = dims[i];
    bx[i] = box[i];
    es[i] = 1;
    if (i > 0) {
      gstr[i - 1] = strides_bytes[i - 1];
      if (gstr[i - 1] % 16 != 0)
        return set_error("TMA global stride %llu B (dim %d) is not a multiple of 16",
                         (unsigned long long)gstr[i - 1], i);
    }
  }
  CUresult r = fn(out, dtype, (cuuint32_t)rank, const_cast<void*>(base),
                  gdim, gstr, bx, es, CU_TENSOR_MAP_INTERLEAVE_NONE, swz,
                  CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS)
    return set_error("cuTensorMapEncodeTiled failed (CUresult %d; rank %d dims %llu,%llu box %u,%u)",
                     (int)r, rank, (unsigned long long)dims[0],
                     (unsigned long long)(rank > 1 ? dims[1] : 0), box[0], rank > 1 ? box[1] : 0);
  return 0;
}

namespace {
struct TmapKey {
  const void* base;
  uint64_t d[3], s[2];
  uint32_t b[3];
  int rank, swz, esize;
  bool operator==(const TmapKey& o) const { return std::memcmp(this, &o, sizeof(TmapKey)) == 0; }
};
struct TmapKeyHash {
  size_t operator()(const TmapKey& k) const {
    size_t h = reinterpret_cast<size_t>(k.base);
    auto mix = [&h](uint64_t v) { h ^= v + 0x9e3779b97f4a7c15ULL + (h << 6) + (h >> 2); };
    for (int i = 0; i < 3; ++i) mix(k.d[i]), mix(k.b[i]);
    mix(k.s[0]), mix(k.s[1]), mix((uint64_t)k.rank), mix((uint64_t)k.swz);
    return h;
  }
};
std::mutex g_tmap_mu;
std::unordered_map<TmapKey, CUtensorMap, TmapKeyHash> g_tmap_cache;
}  // namespace

static int cached_tmap_typed(CUtensorMap* out, const void* base, int rank, const uint64_t* dims,
                             const uint64_t* strides_bytes, const uint32_t* box, CUtensorMapSwizzle swz, int esize);

int cached_tmap_16bit(CUtensorMap* out, const void* base, int rank, const uint64_t* dims,
                      const uint64_t* strides_bytes, const uint32_t* box, CUtensorMapSwizzle swz) {
  return cached_tmap_typed(out, base, rank, dims, strides_bytes, box, swz, 2);
}
int cached_tmap_f32(CUtensorMap* out, const void* base, int rank, const uint64_t* dims,
                    const uint64_t* strides_bytes, const uint32_t* box, CUtensorMapSwizzle swz) {
  return cached_tmap_typed(out, base, rank, dims, strides_bytes, box, swz, 4);
}

static int cached_tmap_typed(CUtensorMap* out, const void* base, int rank, const uint64_t* dims,
                             const uint64_t* strides_bytes, const uint32_t* box, CUtensorMapSwizzle swz, int esize) {
  TmapKey key;
  std::memset(&key, 0, sizeof(key));  // padding bytes take part in the memcmp
  key.base = base, key.rank = rank, key.swz = (int)swz, key.esize = esize;
  for (int i = 0; i < rank && i < 3; ++i) {
    key.d[i] = dims[i];
    key.b[i] = box[i];
    if (i > 0) key.s[i - 1] = strides_bytes[i - 1];
  }
  {
    std::lock_guard<std::mutex> g(g_tmap_mu);
    auto it = g_tmap_cache.find(key);
    if (it != g_tmap_cache.end()) {
      *out = it->second;
      return 0;
    }
  }
  int rc = encode_tmap_typed(out, base, rank, dims, strides_bytes, box, swz,
                             esize == 4 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16);
  if (rc) return rc;
  std::lock_guard<std::mutex> g(g_tmap_mu);
  if (g_tmap_cache.size() > 65536) g_tmap_cache.clear();
  g_tmap_cache.emplace(key, *out);
  return 0;
}

}  // namespace fvit

extern "C" {
int fvit_abi_version(void) { return FVIT_ABI_VERSION; }
const char* fvit_last_error(void) { return fvit::err_buf(); }
int64_t fvit_launch_count(void) { return fvit::g_launches.load(); }
void fvit_reset_launch_count(void) { fvit::g_launches.store(0); }
void fvit_add_launch_count(int64_t n) { fvit::g_launches.fetch_add(n); }
void fvit_set_sm_limit(int32_t n) { fvit::g_sm_limit.store(n > 0 ? n : 0); }
}
