// The forward tile kernel with ALiBi (fwd_sm90.cuh, kAlibi = true), in its own translation unit so that the kernels
// without it (fwd_sm90.cu, fwd_band_sm90.cu) compile exactly as before.
#include "fwd_sm90.cuh"

namespace ba {

int launch_fwd_alibi(int dtype, int D, bool band, const CUtensorMap& tmQ, const CUtensorMap& tmK,
                     const CUtensorMap& tmV, const FwdParams& p, cudaStream_t stream) {
  const bool bf16 = dtype == BA_DTYPE_BF16;
  void (*kern)(CUtensorMap, CUtensorMap, CUtensorMap, FwdParams);
  if (band)
    kern = D == 64 ? (bf16 ? fwd_alibi_kernel<true, 64, true> : fwd_alibi_kernel<false, 64, true>)
                   : (bf16 ? fwd_alibi_kernel<true, 128, true> : fwd_alibi_kernel<false, 128, true>);
  else
    kern = D == 64 ? (bf16 ? fwd_alibi_kernel<true, 64, false> : fwd_alibi_kernel<false, 64, false>)
                   : (bf16 ? fwd_alibi_kernel<true, 128, false> : fwd_alibi_kernel<false, 128, false>);
  const int smem = D == 64 ? FwdLayout<64>::kSmemBytes : FwdLayout<128>::kSmemBytes;
  BA_CHECK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  dim3 grid((p.Sq + kBlockM - 1) / kBlockM, p.H, p.B);
  kern<<<grid, kFwdThreads, smem, stream>>>(tmQ, tmK, tmV, p);
  BA_CHECK_CUDA(cudaGetLastError());
  return BA_OK;
}

}  // namespace ba
