#include "host_util.h"

#include <cstring>
#include <mutex>

namespace ivid {

typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static PFN_encodeTiled get_encode_fn() {
  static PFN_encodeTiled fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres);
    if (e == cudaSuccess && qres == cudaDriverEntryPointSuccess) fn = reinterpret_cast<PFN_encodeTiled>(p);
  });
  if (!fn) throw Error(kErrCuda, "cuTensorMapEncodeTiled is not available from the CUDA driver");
  return fn;
}

CUtensorMap make_tensor_map(CUtensorMapDataType dtype, int rank, void* base, const uint64_t* dims,
                            const uint64_t* strides_bytes, const uint32_t* box, CUtensorMapSwizzle swizzle) {
  CUtensorMap m;
  std::memset(&m, 0, sizeof(m));
  cuuint64_t gdims[5];
  cuuint64_t gstr[4];
  cuuint32_t bx[5];
  cuuint32_t es[5];
  for (int i = 0; i < rank; ++i) {
    gdims[i] = dims[i];
    bx[i] = box[i];
    es[i] = 1;
  }
  for (int i = 0; i + 1 < rank; ++i) gstr[i] = strides_bytes[i];
  CUresult r = get_encode_fn()(&m, dtype, static_cast<cuuint32_t>(rank), base, gdims, gstr, bx, es,
                               CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                               CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    throw Error(kErrCuda, "cuTensorMapEncodeTiled failed with CUresult " + std::to_string(static_cast<int>(r)));
  }
  return m;
}

CUtensorMap make_act_map(const void* base, int N, int H, int W, int C, int TW, int TH, int TN) {
  const uint64_t dims[4] = {static_cast<uint64_t>(C), static_cast<uint64_t>(W), static_cast<uint64_t>(H),
                            static_cast<uint64_t>(N)};
  const uint64_t str[3] = {static_cast<uint64_t>(C) * 2, static_cast<uint64_t>(W) * C * 2,
                           static_cast<uint64_t>(H) * W * C * 2};
  const uint32_t box[4] = {64, static_cast<uint32_t>(TW), static_cast<uint32_t>(TH), static_cast<uint32_t>(TN)};
  return make_tensor_map(CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 4, const_cast<void*>(base), dims, str, box,
                         CU_TENSOR_MAP_SWIZZLE_128B);
}

CUtensorMap make_weight_map(const void* base, int rows, int K, int box_rows) {
  const uint64_t dims[2] = {static_cast<uint64_t>(K), static_cast<uint64_t>(rows)};
  const uint64_t str[1] = {static_cast<uint64_t>(K) * 2};
  const uint32_t box[2] = {64, static_cast<uint32_t>(box_rows)};
  return make_tensor_map(CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, const_cast<void*>(base), dims, str, box,
                         CU_TENSOR_MAP_SWIZZLE_128B);
}

int sm_count() {
  static int n = 0;
  if (n == 0) {
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) return 132;
    cudaDeviceProp prop;
    if (cudaGetDeviceProperties(&prop, dev) != cudaSuccess) return 132;
    n = prop.multiProcessorCount;
  }
  return n;
}

}  // namespace ivid
