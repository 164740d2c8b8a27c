// TEST INFRASTRUCTURE: the marker that keeps the emulation build out of the product, and the host-side model of
// cuTensorMapEncodeTiled that pairs with the TMA model in shim/ptx_sm90.cuh.
#include <cuda.h>
#include <cuda_runtime.h>
#include <string.h>
#include "ptx_sm90.cuh"

extern "C" int pcl_emulated(void) { return 1; }      // contrastiveseg_b200._abi.load refuses a library that exports this

static CUresult emu_encode_tiled(CUtensorMap* m, CUtensorMapDataType dt, cuuint32_t rank, void* base, const cuuint64_t* gdim,
                                 const cuuint64_t* gstride, const cuuint32_t* box, const cuuint32_t*, CUtensorMapInterleave,
                                 CUtensorMapSwizzle sw, CUtensorMapL2promotion, CUtensorMapFloatOOBfill) {
  if (!m || rank != 2 || dt != CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 || sw != CU_TENSOR_MAP_SWIZZLE_128B) return CUDA_ERROR_INVALID_VALUE;
  if (((uintptr_t)base & 15) != 0 || (gstride[0] & 15) != 0 || box[0] * 2 != 128 || box[1] > 256) return CUDA_ERROR_INVALID_VALUE;
  memset(m, 0, sizeof(*m));
  ptx::TmapModel t{(const uint8_t*)base, gdim[1], gstride[0], box[0], box[1], 0x7A3Du};
  memcpy(m, &t, sizeof(t));
  return CUDA_SUCCESS;
}

cudaError_t cudaGetDriverEntryPoint(const char* symbol, void** fn, unsigned long long, cudaDriverEntryPointQueryResult* q) {
  if (symbol && strcmp(symbol, "cuTensorMapEncodeTiled") == 0) {
    *fn = (void*)emu_encode_tiled;
    if (q) *q = cudaDriverEntryPointSuccess;
    return cudaSuccess;
  }
  if (q) *q = cudaDriverEntryPointSymbolNotFound;
  return cudaErrorInvalidValue;
}
