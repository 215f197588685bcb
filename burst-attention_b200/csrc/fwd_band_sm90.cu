// The forward tile kernel with a band's lower edge (fwd_sm90.cuh, kBand = true), in its own translation unit so
// that the kernels without one (fwd_sm90.cu) compile exactly as before.
#include "fwd_sm90.cuh"

namespace ba {

FwdKernel fwd_band_kernel_of(bool bf16, int D, bool bias) { return fwd_chunk_kernel_of<true>(bf16, D, bias); }

}  // namespace ba
