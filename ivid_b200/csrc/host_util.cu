#include "host_util.h"

#include <cmath>
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

static uint64_t elem_bytes(CUtensorMapDataType dtype) {
  return dtype == CU_TENSOR_MAP_DATA_TYPE_UINT8 ? 1 : dtype == CU_TENSOR_MAP_DATA_TYPE_FLOAT32 ? 4 : 2;
}

CUtensorMap make_act_map(const void* base, int N, int H, int W, int C, int TW, int TH, int TN, CUtensorMapDataType dtype,
                         int pitch, int box_c) {
  const uint64_t es = elem_bytes(dtype);
  const uint64_t ld = static_cast<uint64_t>(pitch > 0 ? pitch : C);
  if (box_c <= 0) box_c = static_cast<int>(128 / es);
  const uint64_t dims[4] = {static_cast<uint64_t>(C), static_cast<uint64_t>(W), static_cast<uint64_t>(H),
                            static_cast<uint64_t>(N)};
  const uint64_t str[3] = {ld * es, static_cast<uint64_t>(W) * ld * es, static_cast<uint64_t>(H) * W * ld * es};
  const uint32_t box[4] = {static_cast<uint32_t>(box_c), static_cast<uint32_t>(TW), static_cast<uint32_t>(TH),
                           static_cast<uint32_t>(TN)};
  const uint64_t row = static_cast<uint64_t>(box_c) * es;
  const CUtensorMapSwizzle sw = row == 128 ? CU_TENSOR_MAP_SWIZZLE_128B
                                : row == 64 ? CU_TENSOR_MAP_SWIZZLE_64B
                                : row == 32 ? CU_TENSOR_MAP_SWIZZLE_32B
                                            : CU_TENSOR_MAP_SWIZZLE_NONE;
  return make_tensor_map(dtype, 4, const_cast<void*>(base), dims, str, box, sw);
}

CUtensorMap make_weight_map(const void* base, int rows, int K, int box_rows, CUtensorMapDataType dtype) {
  const uint64_t es = elem_bytes(dtype);
  const uint64_t dims[2] = {static_cast<uint64_t>(K), static_cast<uint64_t>(rows)};
  const uint64_t str[1] = {static_cast<uint64_t>(K) * es};
  const uint32_t box[2] = {static_cast<uint32_t>(128 / es), static_cast<uint32_t>(box_rows)};
  return make_tensor_map(dtype, 2, const_cast<void*>(base), dims, str, box, CU_TENSOR_MAP_SWIZZLE_128B);
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

uint8_t fp8_e4m3_from_float(float v) {
  uint32_t bits;
  std::memcpy(&bits, &v, 4);
  const uint8_t sign = static_cast<uint8_t>((bits >> 24) & 0x80u);
  if ((bits & 0x7FFFFFFFu) > 0x7F800000u) return sign | 0x7F;
  const double a = std::fabs(static_cast<double>(v));
  if (a >= 448.0) return sign | 0x7E;
  if (a < 0.015625) {                                   // below 2^-6: subnormals in steps of 2^-9 (8 rounds up to 2^-6)
    return sign | static_cast<uint8_t>(std::nearbyint(a * 512.0));
  }
  int k;
  const double f = std::frexp(a, &k);                   // a = f * 2^k, f in [0.5, 1): exponent E = k - 1 in [-6, 8]
  int E = k - 1;
  int m = static_cast<int>(std::nearbyint((f * 2.0 - 1.0) * 8.0));   // 3 mantissa bits, ties to even
  if (m == 8) { m = 0; ++E; }
  const int code = ((E + 7) << 3) | m;
  return sign | static_cast<uint8_t>(code > 0x7E ? 0x7E : code);
}

float fp8_e4m3_to_float(uint8_t q) {
  const int e = (q >> 3) & 0xF, m = q & 7;
  if (e == 0xF && m == 7) return std::nanf("");
  const float v = e == 0 ? std::ldexp(static_cast<float>(m), -9) : std::ldexp(1.0f + m / 8.0f, e - 7);
  return (q & 0x80) ? -v : v;
}

int fp8_weight_exponent(float max_abs) {
  if (!(max_abs > 0.f)) return 0;
  int k;
  const double f = std::frexp(static_cast<double>(max_abs), &k);   // max_abs = f * 2^k, f in [0.5, 1)
  // 448 = 0.875 * 2^9: f <= 0.875 scales to f * 2^9 in [256, 448], f > 0.875 to f * 2^8 in (224, 256)
  return (f <= 0.875 ? 9 : 8) - k;
}

}  // namespace ivid
