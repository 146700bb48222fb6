#include "tmap.h"
#include "launchers.h"

#include <mutex>
#include <stdio.h>
#include <string.h>

namespace {
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
EncodeTiledFn g_encode = nullptr;
std::once_flag g_once;
char g_err[512] = {0};

void resolve() {
  void* fn = nullptr;
  cudaDriverEntryPointQueryResult q;
  cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &q);
  if (e == cudaSuccess && q == cudaDriverEntryPointSuccess) g_encode = (EncodeTiledFn)fn;
}
}  // namespace

extern "C" const char* ts_last_error() { return g_err; }

namespace ts {

void set_last_error(const char* msg) {
  strncpy(g_err, msg, sizeof(g_err) - 1);
  g_err[sizeof(g_err) - 1] = 0;
}

int make_tmap_2d_bf16(CUtensorMap* out, const void* base, uint64_t rows, uint64_t cols, uint64_t pitch_elems,
                      uint32_t box_cols, uint32_t box_rows, int swizzle128) {
  std::call_once(g_once, resolve);
  if (!g_encode) { set_last_error("cuTensorMapEncodeTiled entry point not available"); return -10; }
  cuuint64_t dims[2] = {cols, rows};
  cuuint64_t strides[1] = {pitch_elems * 2};
  cuuint32_t box[2] = {box_cols, box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = g_encode(out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(base), dims, strides, box, estr,
                        CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle128 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_NONE,
                        CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    char b[256];
    snprintf(b, sizeof(b), "cuTensorMapEncodeTiled(2d) failed: %d (rows=%llu cols=%llu pitch=%llu box=%ux%u base=%p)", (int)r,
             (unsigned long long)rows, (unsigned long long)cols, (unsigned long long)pitch_elems, box_rows, box_cols, base);
    set_last_error(b);
    return -11;
  }
  return 0;
}

int make_tmap_3d_bf16(CUtensorMap* out, const void* base, uint64_t d0, uint64_t d1, uint64_t d2, uint64_t stride1,
                      uint64_t stride2, uint32_t box0, uint32_t box1, uint32_t box2, int swizzle128) {
  std::call_once(g_once, resolve);
  if (!g_encode) { set_last_error("cuTensorMapEncodeTiled entry point not available"); return -10; }
  cuuint64_t dims[3] = {d0, d1, d2};
  cuuint64_t strides[2] = {stride1 * 2, stride2 * 2};
  cuuint32_t box[3] = {box0, box1, box2};
  cuuint32_t estr[3] = {1, 1, 1};
  CUresult r = g_encode(out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, const_cast<void*>(base), dims, strides, box, estr,
                        CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle128 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_NONE,
                        CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    char b[256];
    snprintf(b, sizeof(b), "cuTensorMapEncodeTiled(3d) failed: %d", (int)r);
    set_last_error(b);
    return -11;
  }
  return 0;
}

int sm_count(int dev) {
  static int cached[64] = {0};
  if (dev < 0 || dev >= 64) dev = 0;
  if (!cached[dev]) {
    int n = 0;
    cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
    cached[dev] = n > 0 ? n : 132;
  }
  return cached[dev];
}

}  // namespace ts
