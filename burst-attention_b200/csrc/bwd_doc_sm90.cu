// The backward tile kernel with packed documents (bwd_sm90.cuh, kDoc = true on the band path), in its own
// translation unit so that the kernels without them (bwd_sm90.cu, bwd_band_sm90.cu, bwd_alibi_sm90.cu) compile
// exactly as before.
#include "bwd_sm90.cuh"

namespace ba {

// the document kernels also stage each Q row's document keys past the other kernels' shared memory
BwdKernel bwd_doc_kernel_of(bool bf16, int D) {
  if (D == 64)
    return {bf16 ? bwd_doc_kernel<true, 64> : bwd_doc_kernel<false, 64>, BwdLayout<64>::kSmemDocBytes};
  return {bf16 ? bwd_doc_kernel<true, 128> : bwd_doc_kernel<false, 128>, BwdLayout<128>::kSmemDocBytes};
}

}  // namespace ba
