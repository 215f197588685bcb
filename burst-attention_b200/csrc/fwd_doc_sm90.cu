// The forward tile kernel with packed documents (fwd_sm90.cuh, kDoc = true on the band path), in its own
// translation unit so that the kernels without them (fwd_sm90.cu, fwd_band_sm90.cu, fwd_alibi_sm90.cu) compile
// exactly as before.
#include "fwd_sm90.cuh"

namespace ba {

FwdKernel fwd_doc_kernel_of(bool bf16, int D) {
  return D == 64 ? (bf16 ? fwd_doc_kernel<true, 64> : fwd_doc_kernel<false, 64>)
                 : (bf16 ? fwd_doc_kernel<true, 128> : fwd_doc_kernel<false, 128>);
}

}  // namespace ba
