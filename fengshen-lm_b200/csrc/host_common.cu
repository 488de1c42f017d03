// fsb200 — library-wide host helpers: error string, device query, TMA tensor-map construction.
#include "host_common.h"

#include <stdarg.h>
#include <stdlib.h>
#include <string.h>

namespace fsb {

static thread_local char g_err[512] = "";

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

int num_sms() {
  static int cached[64] = {0};
  int dev = 0;
  cudaGetDevice(&dev);
  if (dev < 0 || dev >= 64) dev = 0;
  if (cached[dev] == 0) {
    int n = 0;
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) n = 132;
    cached[dev] = n;
  }
  return cached[dev];
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode_fn() {
  static EncodeTiledFn fn = nullptr;
  if (fn) return fn;
  void* p = nullptr;
  cudaDriverEntryPointQueryResult qres;
  cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres);
  if (e != cudaSuccess || qres != cudaDriverEntryPointSuccess || p == nullptr) {
    set_error("cuTensorMapEncodeTiled entry point unavailable: %s", cudaGetErrorString(e));
    return nullptr;
  }
  fn = reinterpret_cast<EncodeTiledFn>(p);
  return fn;
}

// A tensor map is a pure function of (base, rank, dims, strides, box) — element type, swizzle, interleave, L2 promotion and
// out-of-bounds fill are fixed below — and a training step presents the same few hundred operands every iteration (flat parameter
// views, activation buffers the caching allocator hands back at the same addresses). The driver's encode call is memoised in a
// per-thread direct-mapped table: a hit copies 128 bytes. FSB_TMAP_CACHE=0 disables it (A/B measurements).
namespace {
struct TmapKey {
  const void* base;
  uint64_t dims[5];
  uint64_t strides[4];
  uint32_t box[5];
  int32_t rank;
};
struct TmapSlot {
  TmapKey key;
  CUtensorMap map;
  bool valid;
};
constexpr int kTmapSlots = 1024;   // power of two; ~210 KB per calling thread
thread_local TmapSlot* t_tmap_cache = nullptr;

bool tmap_cache_enabled() {
  static const bool on = [] {
    const char* e = getenv("FSB_TMAP_CACHE");
    return !(e && e[0] == '0');
  }();
  return on;
}

uint32_t tmap_hash(const TmapKey& k) {
  uint64_t h = 0xcbf29ce484222325ull;
  auto mix = [&h](uint64_t v) { h = (h ^ v) * 0x100000001b3ull; h ^= h >> 29; };
  mix(reinterpret_cast<uint64_t>(k.base));
  for (int i = 0; i < 5; ++i) mix(k.dims[i]);
  for (int i = 0; i < 4; ++i) mix(k.strides[i]);
  for (int i = 0; i < 5; ++i) mix(k.box[i]);
  mix(static_cast<uint64_t>(k.rank));
  return static_cast<uint32_t>(h ^ (h >> 32)) & (kTmapSlots - 1);
}
}  // namespace

int make_tmap_bf16(CUtensorMap* out, const void* base, int rank, const uint64_t* dims, const uint64_t* strides_bytes,
                   const uint32_t* box) {
  EncodeTiledFn fn = get_encode_fn();
  if (!fn) return FSB_ERR_CUDA;
  if (rank < 1 || rank > 5) {
    set_error("make_tmap_bf16: rank %d outside 1..5", rank);
    return FSB_ERR_INVALID;
  }
  TmapSlot* slot = nullptr;
  TmapKey key;
  if (tmap_cache_enabled()) {
    memset(&key, 0, sizeof(key));
    key.base = base;
    key.rank = rank;
    for (int i = 0; i < rank; ++i) { key.dims[i] = dims[i]; key.box[i] = box[i]; }
    for (int i = 0; i + 1 < rank; ++i) key.strides[i] = strides_bytes[i];
    if (!t_tmap_cache) t_tmap_cache = static_cast<TmapSlot*>(calloc(kTmapSlots, sizeof(TmapSlot)));
    if (t_tmap_cache) {
      slot = &t_tmap_cache[tmap_hash(key)];
      if (slot->valid && memcmp(&slot->key, &key, sizeof(key)) == 0) {
        memcpy(out, &slot->map, sizeof(CUtensorMap));
        return FSB_OK;
      }
    }
  }
  cuuint64_t gdim[5];
  cuuint64_t gstr[4];
  cuuint32_t bdim[5];
  cuuint32_t estr[5];
  for (int i = 0; i < rank; ++i) {
    gdim[i] = dims[i];
    bdim[i] = box[i];
    estr[i] = 1;
  }
  for (int i = 0; i + 1 < rank; ++i) gstr[i] = strides_bytes[i];
  CUresult r = fn(out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, rank, const_cast<void*>(base), gdim, gstr, bdim, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled failed (CUresult %d): rank %d dims [%llu,%llu,%llu] stride0 %llu box [%u,%u]",
              int(r), rank, (unsigned long long)dims[0], (unsigned long long)(rank > 1 ? dims[1] : 0),
              (unsigned long long)(rank > 2 ? dims[2] : 0), (unsigned long long)strides_bytes[0], box[0],
              rank > 1 ? box[1] : 0);
    return FSB_ERR_CUDA;
  }
  if (slot) {
    memcpy(&slot->key, &key, sizeof(key));
    memcpy(&slot->map, out, sizeof(CUtensorMap));
    slot->valid = true;
  }
  return FSB_OK;
}

}  // namespace fsb

extern "C" int fsb_version(void) { return 1000 * 0 + 1; }
extern "C" const char* fsb_last_error(void) { return fsb::g_err; }
extern "C" int fsb_num_sms(void) { return fsb::num_sms(); }
