// fdx_tc_cat.cu -- the tap-GEMM kernel with a two-source A operand (fdx_gemm_cat): six instantiations, TC_KK and TC_KMN
// at each column tile, plain epilogue.  Their own translation unit keeps fdx_tc.cu's set of kernels as it is.
#include "fdx_tc_kernel.cuh"

namespace {

template <int BN, int MODE>
int launch_cat(const CUtensorMap& mA, const CUtensorMap& mB, const CUtensorMap& mA1, const TcDev& d,
               cudaStream_t stream) {
  using Cfg = TcCfg<BN>;
  static bool attr_set = false;
  if (!attr_set) {
    FDX_CUDA(cudaFuncSetAttribute(
        (void (*)(CUtensorMap, CUtensorMap, TcDev, CUtensorMap))fdx_tc_kernel<BN, MODE, EPI_PLAIN, CUtensorMap>,
        cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::kSmemBytes));
    attr_set = true;
  }
  int grid = fdx_num_sms();
  if (grid <= 0) return FDX_ERR_NO_DEVICE;
  if (d.ntiles < grid) grid = d.ntiles;
  fdx_tc_kernel<BN, MODE, EPI_PLAIN, CUtensorMap><<<grid, Cfg::kThreads, Cfg::kSmemBytes, stream>>>(mA, mB, d, mA1);
  fdx_note_kernel(FDX_KERNEL_TC);
  FDX_LAUNCH_CHECK();
  return FDX_OK;
}

template <int MODE>
int launch_cat_mode(int BN, const CUtensorMap& mA, const CUtensorMap& mB, const CUtensorMap& mA1, const TcDev& d,
                    cudaStream_t stream) {
  switch (BN) {
    case 64: return launch_cat<64, MODE>(mA, mB, mA1, d, stream);
    case 128: return launch_cat<128, MODE>(mA, mB, mA1, d, stream);
    case 256: return launch_cat<256, MODE>(mA, mB, mA1, d, stream);
  }
  fdx_set_error("tc: unsupported BN %d", BN);
  return FDX_ERR_UNSUPPORTED;
}

}  // namespace

int fdx_tc_cat_launch(int BN, int mode, const CUtensorMap& mA, const CUtensorMap& mB, const CUtensorMap& mA1,
                      const TcDev& d, cudaStream_t stream) {
  return mode == TC_KK ? launch_cat_mode<TC_KK>(BN, mA, mB, mA1, d, stream)
                       : launch_cat_mode<TC_KMN>(BN, mA, mB, mA1, d, stream);
}
