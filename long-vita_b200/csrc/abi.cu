// C-ABI housekeeping: version, thread-local error text, launch counter, tensor-map encoder.
#include <atomic>
#include <mutex>
#include <string.h>

#include "common.cuh"

namespace lv {

static thread_local char g_err[512] = "";
static std::atomic<int64_t> g_launches{0};

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

void count_launch(int n) { g_launches.fetch_add(n, std::memory_order_relaxed); }

int sm_count() {
  static int cached[64] = {0};
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return 132;
  if (cached[dev] == 0) {
    int n = 0;
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) n = 132;
    cached[dev] = n;
  }
  return cached[dev];
}

int bind_device(const void* ptr) {
  if (ptr == nullptr) return LV_OK;
  cudaPointerAttributes attr;
  cudaError_t e = cudaPointerGetAttributes(&attr, ptr);
  if (e != cudaSuccess) {
    cudaGetLastError();
    set_error("cudaPointerGetAttributes failed: %s", cudaGetErrorString(e));
    return LV_ECUDA;
  }
  if (attr.type != cudaMemoryTypeDevice && attr.type != cudaMemoryTypeManaged) {
    set_error("pointer %p is not device memory", ptr);
    return LV_EINVAL;
  }
  int cur = -1;
  if (cudaGetDevice(&cur) != cudaSuccess || cur != attr.device) {
    e = cudaSetDevice(attr.device);
    if (e != cudaSuccess) {
      set_error("cudaSetDevice(%d) failed: %s", attr.device, cudaGetErrorString(e));
      return LV_ECUDA;
    }
  }
  // cudaSetDevice is lazy about the driver context on some paths; a no-op runtime call binds it
  // (once per host thread and device)
  static thread_local int bound = -1;
  if (bound != attr.device) {
    if (cudaFree(nullptr) != cudaSuccess) cudaGetLastError();
    bound = attr.device;
  }
  return LV_OK;
}

typedef CUresult (*encode_fn_t)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static encode_fn_t get_encode_fn() {
  static encode_fn_t fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<encode_fn_t>(p);
  });
  return fn;
}

int encode_tmap_bf16(CUtensorMap* out, const void* base, int rank, const uint64_t* dims,
                     const uint64_t* strides_bytes, const uint32_t* box, bool swizzle128) {
  encode_fn_t fn = get_encode_fn();
  if (!fn) {
    set_error("cuTensorMapEncodeTiled is not available from the driver");
    return LV_ECUDA;
  }
  if ((reinterpret_cast<uintptr_t>(base) & 15) != 0) {
    set_error("tensor base %p is not 16-byte aligned", base);
    return LV_EINVAL;
  }
  cuuint64_t gdim[5];
  cuuint64_t gstr[5];
  cuuint32_t bx[5];
  cuuint32_t es[5];
  for (int i = 0; i < rank; ++i) {
    gdim[i] = dims[i];
    bx[i] = box[i];
    es[i] = 1;
    if (i > 0) {
      if (strides_bytes[i] % 16 != 0) {
        set_error("tensor stride %llu bytes (dim %d) is not a multiple of 16", (unsigned long long)strides_bytes[i], i);
        return LV_EINVAL;
      }
      gstr[i - 1] = strides_bytes[i];
    }
  }
  CUresult r = fn(out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, (cuuint32_t)rank, const_cast<void*>(base), gdim, gstr, bx,
                  es, CU_TENSOR_MAP_INTERLEAVE_NONE,
                  swizzle128 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_NONE,
                  CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled failed with CUresult %d (rank %d, dims %llu %llu %llu %llu, box %u %u %u %u)",
              (int)r, rank, (unsigned long long)dims[0], (unsigned long long)(rank > 1 ? dims[1] : 0),
              (unsigned long long)(rank > 2 ? dims[2] : 0), (unsigned long long)(rank > 3 ? dims[3] : 0), box[0],
              rank > 1 ? box[1] : 0, rank > 2 ? box[2] : 0, rank > 3 ? box[3] : 0);
    return LV_ECUDA;
  }
  return LV_OK;
}

}  // namespace lv

extern "C" {

int lv_version(void) { return 1 * 1000 + 1; }

const char* lv_last_error(void) { return lv::g_err; }

int64_t lv_launch_count(void) { return lv::g_launches.load(std::memory_order_relaxed); }

}  // extern "C"
