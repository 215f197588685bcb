// The backward tile kernel with a band's lower edge (bwd_sm90.cuh, kBand = true), in its own translation unit so
// that the kernels without one (bwd_sm90.cu) compile exactly as before.
#include "bwd_sm90.cuh"

namespace ba {

int launch_bwd_band(int dtype, int D, const CUtensorMap& tmQ, const CUtensorMap& tmK, const CUtensorMap& tmV,
                    const CUtensorMap& tmDO, const CUtensorMap& tmDQ, const BwdParams& p, cudaStream_t stream) {
  return launch_bwd<true>(dtype, D, tmQ, tmK, tmV, tmDO, tmDQ, p, stream);
}

}  // namespace ba
