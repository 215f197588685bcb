// The backward tile kernel with a band's lower edge (bwd_sm90.cuh, kBand = true), in its own translation unit so
// that the kernels without one (bwd_sm90.cu) compile exactly as before.
#include "bwd_sm90.cuh"

namespace ba {

BwdKernel bwd_band_kernel_of(bool bf16, int D) { return bwd_chunk_kernel_of<true>(bf16, D); }

}  // namespace ba
