// capi.cu — process-wide helpers of libtango_b200.so: error reporting, device query, TMA descriptor encoding.
#include "tng_internal.h"
#include <atomic>
#include <mutex>

namespace tng {

static thread_local char g_err[512] = "";
static std::atomic<uint64_t> g_launches{0};

int set_error(int code, const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
  return code;
}

void count_launch() { g_launches.fetch_add(1, std::memory_order_relaxed); }

int num_sms() {
  static int sms = 0;
  if (sms == 0) {
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) return 1;
    int v = 0;
    if (cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || v <= 0) return 1;
    sms = v;
  }
  return sms;
}

typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static PFN_encodeTiled get_encode() {
  static PFN_encodeTiled fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) == cudaSuccess &&
        qres == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<PFN_encodeTiled>(p);
  });
  return fn;
}

int encode_tmap_bf16(CUtensorMap* out, const void* ptr, int rank, const uint64_t* dims, const uint64_t* strides_bytes,
                     const uint32_t* box) {
  PFN_encodeTiled enc = get_encode();
  if (!enc) return set_error(TNG_ECUDA, "cuTensorMapEncodeTiled unavailable (no CUDA driver / device)");
  if ((reinterpret_cast<uintptr_t>(ptr) & 15) != 0) return set_error(TNG_EINVAL, "TMA base pointer not 16-byte aligned");
  cuuint64_t gdim[5];
  cuuint64_t gstr[4];
  cuuint32_t bx[5];
  cuuint32_t es[5];
  for (int i = 0; i < rank; ++i) {
    gdim[i] = dims[i];
    bx[i] = box[i];
    es[i] = 1;
    if (box[i] == 0 || box[i] > 256) return set_error(TNG_EINVAL, "TMA box dim %d = %u out of range", i, box[i]);
  }
  for (int i = 0; i + 1 < rank; ++i) {
    gstr[i] = strides_bytes[i];
    if (strides_bytes[i] % 16 != 0)
      return set_error(TNG_EINVAL, "TMA stride %d = %llu bytes is not a multiple of 16", i,
                       (unsigned long long)strides_bytes[i]);
  }
  CUresult r = enc(out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, (cuuint32_t)rank, const_cast<void*>(ptr), gdim, gstr, bx, es,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return set_error(TNG_ECUDA, "cuTensorMapEncodeTiled failed: CUresult %d", (int)r);
  return TNG_OK;
}

int encode_tmap_rows_bf16(CUtensorMap* out, const void* ptr, long long ld, long long L, long long batch, uint32_t rows) {
  const uint64_t dims[3] = {(uint64_t)ld, (uint64_t)L, (uint64_t)batch};
  const uint64_t strides[2] = {(uint64_t)ld * 2, (uint64_t)ld * 2 * (uint64_t)L};
  const uint32_t box[3] = {64, rows, 1};
  return encode_tmap_bf16(out, ptr, 3, dims, strides, box);
}

}  // namespace tng

extern "C" int tng_version(void) { return 100; }
extern "C" const char* tng_last_error(void) { return tng::g_err; }
extern "C" uint64_t tng_launch_count(void) { return tng::g_launches.load(); }
