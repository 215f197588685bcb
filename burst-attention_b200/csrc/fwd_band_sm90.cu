// The forward tile kernel with a band's lower edge (fwd_sm90.cuh, kBand = true), in its own translation unit so
// that the kernels without one (fwd_sm90.cu) compile exactly as before.
#include "fwd_sm90.cuh"

namespace ba {

int launch_fwd_band(int dtype, int D, bool bias, const CUtensorMap& tmQ, const CUtensorMap& tmK,
                    const CUtensorMap& tmV, const FwdParams& p, cudaStream_t stream) {
  return launch_fwd<true>(dtype, D, bias, tmQ, tmK, tmV, p, stream);
}

}  // namespace ba
