// Host-side helpers shared by the C-ABI implementation: error handling, TMA tensor-map encoding.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include <stdexcept>
#include <string>

namespace ivid {

struct Error : std::runtime_error {
  int code;
  Error(int c, const std::string& m) : std::runtime_error(m), code(c) {}
};

// status codes of the C ABI (include/ivid_b200.h)
enum : int {
  kOk = 0,
  kErrInvalidArgument = 1,   // maps to Python AssertionError / ValueError
  kErrNotImplemented = 2,    // maps to Python NotImplementedError
  kErrCuda = 3,              // maps to RuntimeError
  kErrState = 4,
};

#define IVID_CHECK_CUDA(expr)                                                                              \
  do {                                                                                                     \
    cudaError_t _e = (expr);                                                                               \
    if (_e != cudaSuccess)                                                                                 \
      throw ::ivid::Error(::ivid::kErrCuda, std::string(#expr) + " failed: " + cudaGetErrorString(_e) +   \
                                                " (" __FILE__ ":" + std::to_string(__LINE__) + ")");       \
  } while (0)

#define IVID_REQUIRE(cond, msg)                                                      \
  do {                                                                               \
    if (!(cond)) throw ::ivid::Error(::ivid::kErrInvalidArgument, std::string(msg)); \
  } while (0)

// cuTensorMapEncodeTiled resolved through the runtime (no link-time dependency on libcuda).
CUtensorMap make_tensor_map(CUtensorMapDataType dtype, int rank, void* base, const uint64_t* dims,
                            const uint64_t* strides_bytes /* rank-1 entries, dim0 is dense */, const uint32_t* box,
                            CUtensorMapSwizzle swizzle);

// NHWC activation [N][H][W][pitch] viewed as (C, W, H, N), C <= pitch (0: pitch = C); box = (box_c channels, TW, TH, TN),
// box_c 0 meaning 128 bytes of channels.  The swizzle spans the box row: 128, 64 or 32 bytes, none at 16.  dtype FLOAT16
// (64-channel box), UINT8 (e4m3 operands, 128-channel box) or FLOAT32 (the conv epilogue's residual and outputs).
CUtensorMap make_act_map(const void* base, int N, int H, int W, int C, int TW, int TH, int TN,
                         CUtensorMapDataType dtype = CU_TENSOR_MAP_DATA_TYPE_FLOAT16, int pitch = 0, int box_c = 0);
// weight matrix [rows][K] (K contiguous); box = (128 bytes of K, box_rows), 128B swizzle; dtype as for make_act_map.
CUtensorMap make_weight_map(const void* base, int rows, int K, int box_rows,
                            CUtensorMapDataType dtype = CU_TENSOR_MAP_DATA_TYPE_FLOAT16);

int sm_count();

// fp32 -> e4m3 (OCP FP8 E4M3FN) on the host: round to nearest even, saturated to +-448, NaN -> 0x7F | sign.  The device
// conversion of the fp8 mode (cvt.rn.satfinite.e4m3x2.f32) gives the same bytes for every non-NaN input.
uint8_t fp8_e4m3_from_float(float v);
float fp8_e4m3_to_float(uint8_t q);
// Power-of-two weight scale of the fp8 mode: the e with max|w| * 2^e in (224, 448]; 0 for max|w| == 0.
int fp8_weight_exponent(float max_abs);

}  // namespace ivid
