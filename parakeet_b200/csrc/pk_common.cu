// Library-wide host plumbing: version, thread-local error string, launch counter, launch setup, TMA descriptor encoding.
#include <stdarg.h>
#include <stdio.h>
#include <string.h>

#include <algorithm>
#include <atomic>
#include <mutex>
#include <vector>

#include "pk_host.h"

namespace pk {

static thread_local char g_err[512] = "";
static std::atomic<long long> g_launches{0};

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

int fail(int code, const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
  return code;
}

void count_launch(int n) { g_launches.fetch_add(n, std::memory_order_relaxed); }

int sm_count() {
  // per device ordinal: a process may drive several devices (grid sizing must follow the CURRENT device)
  static std::atomic<int> cache[64];
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return 132;
  int n = cache[dev].load(std::memory_order_relaxed);
  if (n == 0) {
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) n = 132;
    cache[dev].store(n, std::memory_order_relaxed);
  }
  return n;
}

int prepare_kernel(const void* kernel, int threads, size_t smem, int* resident_ctas) {
  // cudaFuncSetAttribute applies to the current device only, so everything is remembered per device
  struct Prepared {
    const void* kernel;
    int dev, threads;
    size_t smem;
    int resident;   // 0: not queried yet
  };
  static std::mutex mu;
  static std::vector<Prepared> prepared;
  int dev = 0;
  PK_CHECK_CUDA(cudaGetDevice(&dev));
  std::lock_guard<std::mutex> lock(mu);
  Prepared* e = nullptr;
  size_t limit = 0;   // the kernel's raised limit on this device: never lowered, a larger launch prepared earlier relies on it
  for (Prepared& x : prepared) {
    if (x.kernel != kernel || x.dev != dev) continue;
    limit = std::max(limit, x.smem);
    if (x.threads == threads && x.smem == smem) e = &x;
  }
  if (e == nullptr) {
    if (smem > limit)
      PK_CHECK_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem)));
    prepared.push_back({kernel, dev, threads, smem, 0});
    e = &prepared.back();
  }
  if (resident_ctas != nullptr) {
    if (e->resident == 0) {
      int per_sm = 0;
      PK_CHECK_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, threads, smem));
      e->resident = per_sm * sm_count();
    }
    *resident_ctas = e->resident;
  }
  return PK_OK;
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode_fn() {
  static EncodeTiledFn fn = nullptr;
  if (fn == nullptr) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    // resolved through the runtime so the library does not link against libcuda.so (absent on the build box)
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) == cudaSuccess &&
        qres == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(p);
  }
  return fn;
}

int encode_tmap_bf16_3d(CUtensorMap* out, const void* base, uint64_t cols, uint64_t rows, uint64_t batches,
                        uint64_t row_stride_elems, uint64_t batch_stride_elems, uint32_t box_rows) {
  EncodeTiledFn fn = get_encode_fn();
  if (fn == nullptr) return fail(PK_ERR_CUDA, "cuTensorMapEncodeTiled entry point not available (no CUDA driver?)");
  if (batches == 0) batches = 1;
  if (batch_stride_elems == 0) batch_stride_elems = row_stride_elems * rows;  // single-batch operands
  cuuint64_t dims[3] = {cols, rows, batches};
  cuuint64_t strides[2] = {row_stride_elems * 2, batch_stride_elems * 2};  // bytes, dims 1..2
  cuuint32_t box[3] = {64, box_rows, 1};
  cuuint32_t estr[3] = {1, 1, 1};
  if ((strides[0] & 15) || (strides[1] & 15)) return fail(PK_ERR_INVALID_ARG, "TMA strides must be multiples of 16 bytes");
  CUresult r = fn(out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, const_cast<void*>(base), dims, strides, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS)
    return fail(PK_ERR_CUDA, "cuTensorMapEncodeTiled failed (%d): cols=%llu rows=%llu batches=%llu ld=%llu bs=%llu box_rows=%u",
                static_cast<int>(r), (unsigned long long)cols, (unsigned long long)rows, (unsigned long long)batches,
                (unsigned long long)row_stride_elems, (unsigned long long)batch_stride_elems, box_rows);
  return PK_OK;
}

int encode_tmap_f32_3d(CUtensorMap* out, const void* base, uint64_t rows, uint64_t batches, uint64_t batch_stride_elems,
                       uint32_t box_rows) {
  EncodeTiledFn fn = get_encode_fn();
  if (fn == nullptr) return fail(PK_ERR_CUDA, "cuTensorMapEncodeTiled entry point not available (no CUDA driver?)");
  if (batches == 0) batches = 1;
  if (batch_stride_elems == 0) batch_stride_elems = 32 * rows;
  cuuint64_t dims[3] = {32, rows, batches};
  cuuint64_t strides[2] = {32 * 4, batch_stride_elems * 4};  // bytes, dims 1..2
  cuuint32_t box[3] = {32, box_rows, 1};
  cuuint32_t estr[3] = {1, 1, 1};
  if (strides[1] & 15) return fail(PK_ERR_INVALID_ARG, "TMA strides must be multiples of 16 bytes");
  CUresult r = fn(out, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, const_cast<void*>(base), dims, strides, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS)
    return fail(PK_ERR_CUDA, "cuTensorMapEncodeTiled (fp32) failed (%d): rows=%llu batches=%llu bs=%llu box_rows=%u",
                static_cast<int>(r), (unsigned long long)rows, (unsigned long long)batches, (unsigned long long)batch_stride_elems,
                box_rows);
  return PK_OK;
}

int encode_tmap_bf16_planes(CUtensorMap* out, const void* hi, const void* lo, uint64_t cols, uint64_t rows, uint64_t batches,
                            uint64_t row_stride_elems, uint64_t batch_stride_elems, uint32_t box_rows, uint32_t box_cols) {
  EncodeTiledFn fn = get_encode_fn();
  if (fn == nullptr) return fail(PK_ERR_CUDA, "cuTensorMapEncodeTiled entry point not available (no CUDA driver?)");
  if (box_cols != 64 && box_cols != 16) return fail(PK_ERR_INVALID_ARG, "box_cols must be 64 or 16 (got %u)", box_cols);
  const CUtensorMapSwizzle swz = box_cols == 64 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_32B;
  const long long plane = static_cast<const char*>(lo) - static_cast<const char*>(hi);
  if (plane <= 0 || (plane & 15) || plane >= (1ll << 40))
    return fail(PK_ERR_INVALID_ARG, "split planes must come from one allocation, lo after hi at a 16-byte multiple (ops.Split.empty / zeros)");
  if (batches == 0) batches = 1;
  if (batch_stride_elems == 0) batch_stride_elems = row_stride_elems * rows;
  cuuint64_t dims[4] = {cols, rows, batches, 2};
  cuuint64_t strides[3] = {row_stride_elems * 2, batch_stride_elems * 2, static_cast<cuuint64_t>(plane)};
  cuuint32_t box[4] = {box_cols, box_rows, 1, 2};
  cuuint32_t estr[4] = {1, 1, 1, 1};
  if ((strides[0] & 15) || (strides[1] & 15)) return fail(PK_ERR_INVALID_ARG, "TMA strides must be multiples of 16 bytes");
  CUresult r = fn(out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, const_cast<void*>(hi), dims, strides, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, swz, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS)
    return fail(PK_ERR_CUDA, "cuTensorMapEncodeTiled (4-D planes) failed (%d): cols=%llu rows=%llu batches=%llu ld=%llu bs=%llu plane=%lld",
                static_cast<int>(r), (unsigned long long)cols, (unsigned long long)rows, (unsigned long long)batches,
                (unsigned long long)row_stride_elems, (unsigned long long)batch_stride_elems, plane);
  return PK_OK;
}

}  // namespace pk

extern "C" int pk_version(void) { return 100; /* 0.1.0 */ }
extern "C" const char* pk_last_error(void) { return pk::g_err; }
extern "C" int64_t pk_launch_count(void) { return pk::g_launches.load(std::memory_order_relaxed); }
