// Host-side helpers shared by the .cu translation units: error reporting for the C ABI and TMA
// tensor-map encoding through the driver entry point (no link-time dependency on libcuda).
#pragma once
#include <cstdarg>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <utility>
#include <cuda.h>
#include <cuda_runtime.h>

namespace vx {

char* last_error_buf();  // defined in vx_runtime.cu (thread-local 512-byte buffer)

inline int fail(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(last_error_buf(), 512, fmt, ap);
  va_end(ap);
  return 1;
}

#define VX_CHECK_CUDA(expr)                                                                      \
  do {                                                                                           \
    cudaError_t _e = (expr);                                                                     \
    if (_e != cudaSuccess) return vx::fail("%s:%d %s -> %s", __FILE__, __LINE__, #expr, cudaGetErrorString(_e)); \
  } while (0)

#define VX_REQUIRE(cond, ...)                 \
  do {                                        \
    if (!(cond)) return vx::fail(__VA_ARGS__); \
  } while (0)

typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
PFN_encodeTiled get_encode_tiled();  // vx_runtime.cu

int device_sms();  // multiprocessors of the current device (vx_runtime.cu)

// bf16 tensor map of rank `rank`: dims[i] elements, strides_bytes[i-1] for i>=1, box[i] elements.
// estrides (optional): traversal stride per dimension (1..8): the box then covers box[i] tensor elements of which every
// estrides[i]-th is loaded, i.e. box[i] / estrides[i] elements land in shared memory (the stride-2 convolutions).
// dtype: CU_TENSOR_MAP_DATA_TYPE_UINT8 for the e4m3 operands of vx_gemm_fp8 (TMA only moves bytes).
inline int make_tmap_bf16(CUtensorMap* m, const void* base, int rank, const uint64_t* dims,
                          const uint64_t* strides_bytes, const uint32_t* box, CUtensorMapSwizzle swz,
                          const uint32_t* estrides = nullptr,
                          CUtensorMapDataType dtype = CU_TENSOR_MAP_DATA_TYPE_BFLOAT16) {
  PFN_encodeTiled enc = get_encode_tiled();
  if (!enc) return fail("cuTensorMapEncodeTiled entry point unavailable");
  cuuint64_t gd[5];
  cuuint64_t gs[4];
  cuuint32_t bx[5];
  cuuint32_t es[5];
  for (int i = 0; i < rank; ++i) {
    gd[i] = dims[i];
    bx[i] = box[i];
    es[i] = estrides ? estrides[i] : 1;
    if (i) gs[i - 1] = strides_bytes[i - 1];
  }
  CUresult r = enc(m, dtype, (cuuint32_t)rank, const_cast<void*>(base), gd, gs, bx, es,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, swz, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS)
    return fail("cuTensorMapEncodeTiled failed: %d (rank %d dims %llu,%llu box %u,%u)", (int)r, rank,
                (unsigned long long)dims[0], (unsigned long long)(rank > 1 ? dims[1] : 0), box[0], rank > 1 ? box[1] : 0);
  return 0;
}

// Programmatic dependent launch: every hot-path kernel starts with `griddepcontrol.launch_dependents` (its successor may
// be scheduled as soon as all of this grid's CTAs have started) and runs `griddepcontrol.wait` before its first access to
// global memory (which returns once the predecessor grid has completed and flushed).  Launched through launch_k with the
// programmatic-stream-serialization attribute, the successor's launch latency and prologue (barrier init,
// tensor-map prefetch, parameter staging) overlap the predecessor's tail, in eager streams and as
// programmatic edges under CUDA-graph capture.  VX_PDL=0 launches with full stream serialisation (A/B switch, read once).
bool pdl_enabled();  // vx_runtime.cu

template <typename... KArgs, typename... Args>
inline cudaError_t launch_k(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, Args&&... args) {
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = pdl_enabled() ? 1 : 0;
  return cudaLaunchKernelEx(&cfg, kern, std::forward<Args>(args)...);
}

}  // namespace vx
