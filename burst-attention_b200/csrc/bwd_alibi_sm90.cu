// The backward tile kernel with ALiBi (bwd_sm90.cuh, kAlibi = true), in its own translation unit so that the kernels
// without it (bwd_sm90.cu, bwd_band_sm90.cu) compile exactly as before.
#include "bwd_sm90.cuh"

namespace ba {

int launch_bwd_alibi(int dtype, int D, bool band, const CUtensorMap& tmQ, const CUtensorMap& tmK,
                     const CUtensorMap& tmV, const CUtensorMap& tmDO, const CUtensorMap& tmDQ, const BwdParams& p,
                     cudaStream_t stream) {
  const bool bf16 = dtype == BA_DTYPE_BF16;
  void (*kern)(CUtensorMap, CUtensorMap, CUtensorMap, CUtensorMap, CUtensorMap, BwdParams);
  if (band)
    kern = D == 64 ? (bf16 ? bwd_alibi_kernel<true, 64, true> : bwd_alibi_kernel<false, 64, true>)
                   : (bf16 ? bwd_alibi_kernel<true, 128, true> : bwd_alibi_kernel<false, 128, true>);
  else
    kern = D == 64 ? (bf16 ? bwd_alibi_kernel<true, 64, false> : bwd_alibi_kernel<false, 64, false>)
                   : (bf16 ? bwd_alibi_kernel<true, 128, false> : bwd_alibi_kernel<false, 128, false>);
  const int smem = D == 64 ? BwdLayout<64>::kSmemBytes : BwdLayout<128>::kSmemBytes;
  BA_CHECK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  dim3 grid((p.Sk + kBwdN - 1) / kBwdN, p.H / p.G, p.B);  // one CTA per (key block, K/V head, batch)
  kern<<<grid, kBwdThreads, smem, stream>>>(tmQ, tmK, tmV, tmDO, tmDQ, p);
  BA_CHECK_CUDA(cudaGetLastError());
  return BA_OK;
}

}  // namespace ba
