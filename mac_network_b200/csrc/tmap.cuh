// CUtensorMap construction without linking libcuda: cuTensorMapEncodeTiled is fetched through the runtime's
// driver-entry-point query.  A small cache keyed by (pointer, geometry) keeps repeated calls off the driver.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <mutex>
#include <string.h>
#include "common.cuh"

namespace mac {

typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

inline PFN_encodeTiled get_encode_fn() {
  static PFN_encodeTiled fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<PFN_encodeTiled>(p);
  });
  return fn;
}

struct TmapKey {
  const void* base;
  int dtype, swizzle;
  uint64_t rows, cols, row_stride_bytes;
  uint32_t box_rows, box_cols;
  bool operator==(const TmapKey& o) const { return memcmp(this, &o, sizeof(TmapKey)) == 0; }
};

// 2-D row-major tensor [rows, cols] (cols contiguous), box = [box_rows, box_cols].  dtype: 0 fp32, 1 bf16, 2 one byte (e4m3).
// swizzle: 0 none, 1 128B.  Returns MAC_OK or MAC_ERR_ARCH / MAC_ERR_INVALID.
inline int make_tmap_2d(CUtensorMap* out, const void* base, int dtype, uint64_t rows, uint64_t cols,
                        uint64_t row_stride_bytes, uint32_t box_rows, uint32_t box_cols, int swizzle) {
  // direct-mapped cache of 2048 descriptors (a training step of netLength 12 uses a few hundred distinct (pointer, geometry)
  // pairs; the 64-entry linear cache of round 1 thrashed there and every launch paid a cuTensorMapEncodeTiled)
  constexpr int NSLOT = 2048;
  static std::mutex mu;
  static TmapKey* keys = new TmapKey[NSLOT]();
  static CUtensorMap* maps = new CUtensorMap[NSLOT];
  static bool* used = new bool[NSLOT]();
  TmapKey k;
  memset(&k, 0, sizeof(k));
  k.base = base; k.dtype = dtype; k.swizzle = swizzle; k.rows = rows; k.cols = cols;
  k.row_stride_bytes = row_stride_bytes; k.box_rows = box_rows; k.box_cols = box_cols;
  uint64_t h = 1469598103934665603ull;
  {
    const unsigned char* kp = reinterpret_cast<const unsigned char*>(&k);
    for (size_t i = 0; i < sizeof(TmapKey); ++i) h = (h ^ kp[i]) * 1099511628211ull;
  }
  const int slot = (int)(h % NSLOT);
  {
    std::lock_guard<std::mutex> g(mu);
    if (used[slot] && keys[slot] == k) { *out = maps[slot]; return MAC_OK; }
  }
  PFN_encodeTiled enc = get_encode_fn();
  if (!enc) return MAC_ERR_ARCH;
  const cuuint64_t gdim[2] = {cols, rows};
  const cuuint64_t gstride[1] = {row_stride_bytes};
  const cuuint32_t box[2] = {box_cols, box_rows};
  const cuuint32_t estr[2] = {1, 1};
  const CUtensorMapDataType dt = dtype == 0   ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32
                                 : dtype == 1 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16
                                              : CU_TENSOR_MAP_DATA_TYPE_UINT8;
  const CUtensorMapSwizzle sw = swizzle ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_NONE;
  CUresult r = enc(out, dt, 2, const_cast<void*>(base), gdim, gstride, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, sw,
                   CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return MAC_ERR_INVALID;
  {
    std::lock_guard<std::mutex> g(mu);
    keys[slot] = k;
    maps[slot] = *out;
    used[slot] = true;
  }
  return MAC_OK;
}

}  // namespace mac
