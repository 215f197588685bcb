// The backward tile kernel with ALiBi (bwd_sm90.cuh, kAlibi = true), in its own translation unit so that the kernels
// without it (bwd_sm90.cu, bwd_band_sm90.cu) compile exactly as before.
#include "bwd_sm90.cuh"

namespace ba {

BwdKernel bwd_alibi_kernel_of(bool bf16, int D, bool band) {
  if (D == 64)
    return {band ? (bf16 ? bwd_alibi_kernel<true, 64, true> : bwd_alibi_kernel<false, 64, true>)
                 : (bf16 ? bwd_alibi_kernel<true, 64, false> : bwd_alibi_kernel<false, 64, false>),
            BwdLayout<64>::kSmemBytes};
  return {band ? (bf16 ? bwd_alibi_kernel<true, 128, true> : bwd_alibi_kernel<false, 128, true>)
               : (bf16 ? bwd_alibi_kernel<true, 128, false> : bwd_alibi_kernel<false, 128, false>),
          BwdLayout<128>::kSmemBytes};
}

}  // namespace ba
