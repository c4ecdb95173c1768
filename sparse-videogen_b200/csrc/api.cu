// Library-level entry points: version, last error, device check, TMA descriptor encoding.
#include <string.h>

#include "../../include/svgb200.h"
#include "host_common.h"

namespace svgb {

static thread_local char g_err[512] = "";

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}
const char* get_error() { return g_err; }

typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*,
                                    const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                    const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                    CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static PFN_encodeTiled get_encode() {
  static PFN_encodeTiled fn = nullptr;
  if (fn) return fn;
  void* p = nullptr;
  cudaDriverEntryPointQueryResult qres;
  cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres);
  if (e != cudaSuccess || qres != cudaDriverEntryPointSuccess || !p) return nullptr;
  fn = reinterpret_cast<PFN_encodeTiled>(p);
  return fn;
}

// rank-D TMA descriptor of 16-bit or e4m3 rows: dims[0] = D elements per row, byte strides of dims 1.., box of one
// 128-byte panel x box_rows rows x 1 ...
static int encode_rows(CUtensorMap* map, const void* base, int dtype, int rank, const cuuint64_t* dims,
                       const long long* strides_elems, int box_rows) {
  PFN_encodeTiled enc = get_encode();
  SVGB_REQUIRE(enc != nullptr, "cuTensorMapEncodeTiled unavailable (no CUDA driver?)");
  SVGB_REQUIRE((reinterpret_cast<uintptr_t>(base) & 15) == 0, "tensor base must be 16-byte aligned");
  const int eb = dtype == SVGB_E4M3 ? 1 : 2;  // bytes per element
  cuuint64_t strides[3];
  for (int i = 0; i + 1 < rank; ++i) {
    SVGB_REQUIRE((strides_elems[i] * eb) % 16 == 0, "strides must be multiples of 16 bytes");
    strides[i] = static_cast<cuuint64_t>(strides_elems[i]) * eb;
  }
  cuuint32_t box[4] = {static_cast<cuuint32_t>(128 / eb), static_cast<cuuint32_t>(box_rows), 1, 1};  // 128-byte rows
  cuuint32_t estr[4] = {1, 1, 1, 1};
  CUresult r = enc(map, dtype == SVGB_BF16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16
                        : dtype == SVGB_F16 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16
                                            : CU_TENSOR_MAP_DATA_TYPE_UINT8,
                   rank, const_cast<void*>(base), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                   CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  SVGB_REQUIRE(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled failed with CUresult %d", (int)r);
  return 0;
}

int encode_tmap_hsd(CUtensorMap* map, const void* base, int dtype, int BH, int S, int D,
                    long long row_stride_elems, long long head_stride_elems, int box_rows) {
  const cuuint64_t dims[3] = {static_cast<cuuint64_t>(D), static_cast<cuuint64_t>(S), static_cast<cuuint64_t>(BH)};
  const long long st[2] = {row_stride_elems, head_stride_elems};
  return encode_rows(map, base, dtype, 3, dims, st, box_rows);
}

int encode_tmap_bhsd(CUtensorMap* map, const void* base, int dtype, int B, int H, int S, int D, Strides st) {
  const cuuint64_t dims[4] = {static_cast<cuuint64_t>(D), static_cast<cuuint64_t>(S), static_cast<cuuint64_t>(H),
                              static_cast<cuuint64_t>(B)};
  const long long s[3] = {st.r, st.h, st.b};
  return encode_rows(map, base, dtype, 4, dims, s, 128);
}

int encode_tmap_scale_rows(CUtensorMap* map, const float* base, int num_blocks, int H, int block_rows) {
  PFN_encodeTiled enc = get_encode();
  SVGB_REQUIRE(enc != nullptr, "cuTensorMapEncodeTiled unavailable (no CUDA driver?)");
  SVGB_REQUIRE((reinterpret_cast<uintptr_t>(base) & 15) == 0 && block_rows % 4 == 0,
               "per-row scales must be 16-byte aligned with block_rows a multiple of 4");
  const cuuint64_t dims[3] = {static_cast<cuuint64_t>(block_rows), static_cast<cuuint64_t>(H),
                              static_cast<cuuint64_t>(num_blocks)};
  const cuuint64_t strides[2] = {static_cast<cuuint64_t>(block_rows) * 4, static_cast<cuuint64_t>(block_rows) * H * 4};
  const cuuint32_t box[3] = {128, 1, 1}, estr[3] = {1, 1, 1};
  CUresult r = enc(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, const_cast<float*>(base), dims, strides, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  SVGB_REQUIRE(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled failed with CUresult %d", (int)r);
  return 0;
}

}  // namespace svgb

extern "C" {

int svgb_version(void) { return 100; }

const char* svgb_last_error(void) { return svgb::get_error(); }

int svgb_device_check(int* sm_major, int* sm_minor, int* num_sms) {
  int dev = 0;
  SVGB_CUDA(cudaGetDevice(&dev));
  cudaDeviceProp prop;
  SVGB_CUDA(cudaGetDeviceProperties(&prop, dev));
  if (sm_major) *sm_major = prop.major;
  if (sm_minor) *sm_minor = prop.minor;
  if (num_sms) *num_sms = prop.multiProcessorCount;
  SVGB_REQUIRE(prop.major == 9 && prop.minor == 0, "svgb200 needs an sm_90 (H100) device, found sm_%d%d",
               prop.major, prop.minor);
  return 0;
}

}  // extern "C"
