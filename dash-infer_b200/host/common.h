// allspark-shaped host layer for the b200spark hot path — common enums and helpers.
// Mirrors the surface (names, values, meaning) of the reference so the operator shims read like the originals:
//   AsStatus            csrc/interface/allspark_check.h:61-85
//   DataType/DeviceType csrc/proto/allspark.proto:35-76
//   UnaryType/BinaryType csrc/proto/allspark.proto (UnaryType {0 none,1 tanh,2 gelu_erf,3 gelu_tanh,4 relu,5 silu,6 sigmoid})
//   AsCacheMode         csrc/interface/allspark.h (AsCacheDefault / AsCacheQuantI8 / AsCacheQuantU4)
#pragma once
#include <cstddef>
#include <cstdint>
#include <cstdio>
#include <stdexcept>
#include <string>

namespace allspark {

enum class AsStatus : int {
  ALLSPARK_SUCCESS = 0,
  ALLSPARK_UNKNOWN_ERROR = 1,
  ALLSPARK_PARAM_ERROR = 2,
  ALLSPARK_IO_ERROR = 3,
  ALLSPARK_MEMORY_ERROR = 4,
  ALLSPARK_RUNTIME_ERROR = 5,
  ALLSPARK_EXCEED_LIMIT_ERROR = 7,
  ALLSPARK_INVALID_CALL_ERROR = 8,
  ALLSPARK_CACHE_MEMORY_OUT = 11,
};

enum DataType : int {
  DATATYPE_UNDEFINED = 0,
  FLOAT32 = 1,
  FLOAT16 = 2,
  INT8 = 3,
  INT16 = 4,
  INT32 = 5,
  INT64 = 6,
  BFLOAT16 = 9,
  UINT8 = 10,
  POINTER = 20,
};

enum DeviceType : int { DEVICETYPE_UNDEFINED = 0, CPU = 1, CUDA = 2 };
enum DataMode : int { DENSE = 0 };
enum UnaryType : int { UNARYTYPE_UNDEFINED = 0, TANH = 1, GELU_ERF = 2, GELU_TANH = 3, RELU = 4, SILU = 5, SIGMOID = 6 };
enum BinaryType : int { BINARYTYPE_UNDEFINED = 0, ADD = 1, MUL = 2 };
// AsCacheQuantFP8 is an extension (not in the reference's enum): the fp8-e4m3 span cache B2_KV_FP8, head 128 only
enum class AsCacheMode : int { AsCacheDefault = 0, AsCacheQuantI8 = 1, AsCacheQuantU4 = 2, AsCacheQuantFP8 = 3 };

inline size_t SizeofType(DataType t) {
  switch (t) {
    case POINTER: case INT64: return 8;
    case FLOAT32: case INT32: return 4;
    case FLOAT16: case BFLOAT16: case INT16: return 2;
    case INT8: case UINT8: return 1;
    default: return 0;
  }
}

class AsException : public std::runtime_error {
 public:
  explicit AsException(const std::string& m) : std::runtime_error(m) {}
};

#define AS_CHECK_STATUS(expr)                                                   \
  do {                                                                          \
    ::allspark::AsStatus _s = (expr);                                           \
    if (_s != ::allspark::AsStatus::ALLSPARK_SUCCESS) return _s;                \
  } while (0)

#define AS_LOG_ERROR(...)                 \
  do {                                    \
    std::fprintf(stderr, "[allspark_b200] " __VA_ARGS__); \
    std::fprintf(stderr, "\n");           \
  } while (0)

// b2_status -> AsStatus (include/b200spark.h status codes)
inline AsStatus FromB2(int st) {
  switch (st) {
    case 0: return AsStatus::ALLSPARK_SUCCESS;
    case 3: return AsStatus::ALLSPARK_PARAM_ERROR;
    case 4: return AsStatus::ALLSPARK_EXCEED_LIMIT_ERROR;
    case 6: return AsStatus::ALLSPARK_PARAM_ERROR;  // unsupported configuration
    default: return AsStatus::ALLSPARK_RUNTIME_ERROR;
  }
}

}  // namespace allspark
