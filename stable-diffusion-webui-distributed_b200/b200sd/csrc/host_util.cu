// host_util.cu — tensor-map encoding through the driver entry point, version string.
#include "tc_common.cuh"

namespace b200sd {

PFN_encodeTiled get_encode_tiled() {
  // function-local static with an initialiser: C++11 makes this thread-safe (one LocalGPUWorker thread per device may
  // reach it at the same time)
  static const PFN_encodeTiled fn = []() -> PFN_encodeTiled {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) == cudaSuccess &&
        qres == cudaDriverEntryPointSuccess)
      return reinterpret_cast<PFN_encodeTiled>(p);
    return nullptr;
  }();
  return fn;
}

static int make_tmap(CUtensorMap* out, const void* base, int rank, const uint64_t* dims, const uint64_t* strides_bytes,
                     const uint32_t* box, const uint32_t* elem_strides, CUtensorMapSwizzle swizzle) {
  PFN_encodeTiled enc = get_encode_tiled();
  if (!enc) return B200SD_ERR_TMAP;
  cuuint64_t gdim[5];
  cuuint64_t gstr[4];
  cuuint32_t bx[5], es[5];
  for (int i = 0; i < rank; ++i) {
    gdim[i] = dims[i];
    bx[i] = box[i];
    es[i] = elem_strides[i];
  }
  for (int i = 0; i + 1 < rank; ++i) {
    gstr[i] = strides_bytes[i];
    if (gstr[i] % 16 != 0) return B200SD_ERR_INVALID;
  }
  // fp16 and bf16 are both 2-byte types: the tensor map only moves bytes
  CUresult r = enc(out, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, static_cast<cuuint32_t>(rank), const_cast<void*>(base), gdim,
                   gstr, bx, es, CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? B200SD_OK : B200SD_ERR_TMAP;
}

int make_tmap_sw128(CUtensorMap* out, const void* base, int rank, const uint64_t* dims, const uint64_t* strides_bytes,
                    const uint32_t* box, const uint32_t* elem_strides) {
  return make_tmap(out, base, rank, dims, strides_bytes, box, elem_strides, CU_TENSOR_MAP_SWIZZLE_128B);
}

int make_tmap_sw64(CUtensorMap* out, const void* base, int rank, const uint64_t* dims, const uint64_t* strides_bytes,
                   const uint32_t* box, const uint32_t* elem_strides) {
  return make_tmap(out, base, rank, dims, strides_bytes, box, elem_strides, CU_TENSOR_MAP_SWIZZLE_64B);
}

}  // namespace b200sd

extern "C" const char* b200sd_version(void) { return "b200sd 0.8 sm_90a"; }
