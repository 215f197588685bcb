// The forward tile kernel with ALiBi (fwd_sm90.cuh, kAlibi = true), in its own translation unit so that the kernels
// without it (fwd_sm90.cu, fwd_band_sm90.cu) compile exactly as before.
#include "fwd_sm90.cuh"

namespace ba {

FwdKernel fwd_alibi_kernel_of(bool bf16, int D, bool band) {
  if (band)
    return D == 64 ? (bf16 ? fwd_alibi_kernel<true, 64, true> : fwd_alibi_kernel<false, 64, true>)
                   : (bf16 ? fwd_alibi_kernel<true, 128, true> : fwd_alibi_kernel<false, 128, true>);
  return D == 64 ? (bf16 ? fwd_alibi_kernel<true, 64, false> : fwd_alibi_kernel<false, 64, false>)
                 : (bf16 ? fwd_alibi_kernel<true, 128, false> : fwd_alibi_kernel<false, 128, false>);
}

}  // namespace ba
