// The forward tile kernel with packed documents (fwd_sm90.cuh, kDoc = true on the band path), in its own
// translation unit so that the kernels without them (fwd_sm90.cu, fwd_band_sm90.cu, fwd_alibi_sm90.cu) compile
// exactly as before.
#include "fwd_sm90.cuh"

namespace ba {

int launch_fwd_doc(int dtype, int D, const CUtensorMap& tmQ, const CUtensorMap& tmK, const CUtensorMap& tmV,
                   const FwdParams& p, cudaStream_t stream) {
  const bool bf16 = dtype == BA_DTYPE_BF16;
  void (*kern)(CUtensorMap, CUtensorMap, CUtensorMap, FwdParams) =
      D == 64 ? (bf16 ? fwd_doc_kernel<true, 64> : fwd_doc_kernel<false, 64>)
              : (bf16 ? fwd_doc_kernel<true, 128> : fwd_doc_kernel<false, 128>);
  const int smem = D == 64 ? FwdLayout<64>::kSmemBytes : FwdLayout<128>::kSmemBytes;
  BA_CHECK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  dim3 grid((p.Sq + kBlockM - 1) / kBlockM, p.H, p.B);
  kern<<<grid, kFwdThreads, smem, stream>>>(tmQ, tmK, tmV, p);
  BA_CHECK_CUDA(cudaGetLastError());
  return BA_OK;
}

}  // namespace ba
