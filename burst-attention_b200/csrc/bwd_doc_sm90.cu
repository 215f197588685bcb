// The backward tile kernel with packed documents (bwd_sm90.cuh, kDoc = true on the band path), in its own
// translation unit so that the kernels without them (bwd_sm90.cu, bwd_band_sm90.cu, bwd_alibi_sm90.cu) compile
// exactly as before.
#include "bwd_sm90.cuh"

namespace ba {

int launch_bwd_doc(int dtype, int D, const CUtensorMap& tmQ, const CUtensorMap& tmK, const CUtensorMap& tmV,
                   const CUtensorMap& tmDO, const CUtensorMap& tmDQ, const BwdParams& p, cudaStream_t stream) {
  const bool bf16 = dtype == BA_DTYPE_BF16;
  void (*kern)(CUtensorMap, CUtensorMap, CUtensorMap, CUtensorMap, CUtensorMap, BwdParams) =
      D == 64 ? (bf16 ? bwd_doc_kernel<true, 64> : bwd_doc_kernel<false, 64>)
              : (bf16 ? bwd_doc_kernel<true, 128> : bwd_doc_kernel<false, 128>);
  const int smem = D == 64 ? BwdLayout<64>::kSmemDocBytes : BwdLayout<128>::kSmemDocBytes;
  BA_CHECK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  dim3 grid((p.Sk + kBwdN - 1) / kBwdN, p.H / p.G, p.B);  // one CTA per (key block, K/V head, batch)
  kern<<<grid, kBwdThreads, smem, stream>>>(tmQ, tmK, tmV, tmDO, tmDQ, p);
  BA_CHECK_CUDA(cudaGetLastError());
  return BA_OK;
}

}  // namespace ba
