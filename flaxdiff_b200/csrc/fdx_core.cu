// fdx_core.cu -- error plumbing, device query and TMA descriptor encoding.
#include "fdx_common.cuh"
#include "../../include/fdx.h"
#include <stdarg.h>
#include <string.h>
#include <mutex>

namespace {
thread_local char g_err[512] = "";
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*,
                                  const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                  const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
EncodeTiledFn g_encode = nullptr;
std::once_flag g_encode_once;
int g_sms = -1;
unsigned long long g_launches = 0;
int g_last_kind = -1;
}  // namespace

void fdx_count_launch() { ++g_launches; }
void fdx_note_kernel(int kind) { g_last_kind = kind; }

void fdx_set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

int fdx_check_cuda(cudaError_t e, const char* what) {
  if (e == cudaSuccess) return FDX_OK;
  fdx_set_error("CUDA error %d (%s) at %s", (int)e, cudaGetErrorString(e), what);
  return FDX_ERR_CUDA;
}

int fdx_num_sms() {
  if (g_sms > 0) return g_sms;
  int dev = 0, sms = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return -1;
  if (cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess) return -1;
  g_sms = sms;
  return sms;
}

int fdx_make_tmap_bf16(CUtensorMap* map, const void* base, int rank, const uint64_t* dims,
                       const uint64_t* strides_bytes, const uint32_t* box,
                       const uint32_t* elem_strides, int swizzle_128b) {
  std::call_once(g_encode_once, []() {
    void* fn = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres) ==
            cudaSuccess &&
        qres == cudaDriverEntryPointSuccess)
      g_encode = reinterpret_cast<EncodeTiledFn>(fn);
  });
  if (!g_encode) {
    fdx_set_error("cuTensorMapEncodeTiled unavailable (no CUDA driver?)");
    return FDX_ERR_NO_DEVICE;
  }
  cuuint64_t gd[5], gs[4];
  cuuint32_t bx[5], es[5];
  for (int i = 0; i < rank; ++i) {
    gd[i] = dims[i];
    bx[i] = box[i];
    es[i] = elem_strides[i];
    if (box[i] == 0 || box[i] > 256) {
      fdx_set_error("tmap: box[%d]=%u out of range", i, box[i]);
      return FDX_ERR_INVALID_ARG;
    }
  }
  for (int i = 0; i < rank - 1; ++i) {
    gs[i] = strides_bytes[i];
    if (gs[i] % 16 != 0) {
      fdx_set_error("tmap: stride[%d]=%llu bytes is not a multiple of 16", i + 1,
                    (unsigned long long)gs[i]);
      return FDX_ERR_INVALID_ARG;
    }
  }
  if ((reinterpret_cast<uintptr_t>(base) & 15) != 0) {
    fdx_set_error("tmap: base pointer not 16-byte aligned");
    return FDX_ERR_INVALID_ARG;
  }
  CUresult r = g_encode(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, (cuuint32_t)rank,
                        const_cast<void*>(base), gd, gs, bx, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
                        swizzle_128b ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_NONE,
                        CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    fdx_set_error(
        "cuTensorMapEncodeTiled failed (%d): rank=%d dims=(%llu,%llu,%llu,%llu) box=(%u,%u,%u,%u)",
        (int)r, rank, (unsigned long long)gd[0], (unsigned long long)(rank > 1 ? gd[1] : 0),
        (unsigned long long)(rank > 2 ? gd[2] : 0), (unsigned long long)(rank > 3 ? gd[3] : 0),
        bx[0], rank > 1 ? bx[1] : 0, rank > 2 ? bx[2] : 0, rank > 3 ? bx[3] : 0);
    return FDX_ERR_CUDA;
  }
  return FDX_OK;
}

extern "C" {
const char* fdx_last_error(void) { return g_err; }
int fdx_version(void) { return 100; }
int fdx_device_sm_count(void) { return fdx_num_sms(); }
unsigned long long fdx_launch_count(void) { return g_launches; }
int fdx_last_kernel_kind(void) { return g_last_kind; }
const char* fdx_kernel_kind_name(int kind) {
  switch (kind) {
    case FDX_KERNEL_TC: return "fdx_tc_kernel";
    case FDX_KERNEL_TCT: return "fdx_tct_kernel";
    case FDX_KERNEL_WGRAD9: return "fdx_wgrad9_kernel";
    case FDX_KERNEL_ATTN_FWD: return "fdx_attn_fwd_kernel";
    case FDX_KERNEL_ATTN_BWD: return "fdx_attn_bwd_kernel";
  }
  return "other";
}
}
