// Self tests of the sm_90a building blocks used by the attention kernels
// (called from tests/ only, through ba_selftest): they isolate the TMA box /
// swizzle layout, the K-major and MN-major shared-memory descriptors, the
// wgmma accumulator fragment and the register-A (RS) form of wgmma, so a failing
// attention parity test can be traced to one assumption.
#include "burst_attn_b200_selftest.h"
#include "host_common.h"
#include "sm90_ptx.cuh"

namespace ba {

constexpr int kStTile = 128 * 128 * 2;  // 32 KiB
constexpr int kStBox = kStTile / 2;
constexpr int kStSmem = 2 * kStTile + 1024 + 64;

// One warpgroup; out[128,128] fp32 is computed as two m64n128 halves (rows 64 hm ..).
// mode 0: out = A * B^T (SS, both K-major)      mode 1: out = A (registers) * B (RS, B MN-major [k][n])
// mode 3: out = A^T * B (SS, A MN-major [k][m], B MN-major [k][n])   -- used by the backward's dQ
// mode 2: raw dump of the first TMA box of A
template <bool kBF16>
__global__ void __launch_bounds__(128, 1)
selftest_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                const uint16_t* __restrict__ a_raw, void* __restrict__ out, int mode) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sA = smem;
  uint8_t* sB = smem + kStTile;
  uint64_t* bar_load = reinterpret_cast<uint64_t*>(sB + kStTile);
  const int t = threadIdx.x, w = t >> 5, lane = t & 31, g = lane >> 2, q = lane & 3;

  if (t == 0) {
    mbar_init(bar_load, 1);
    fence_mbar_init();
  }
  __syncthreads();
  if (t == 0) {
    mbar_arrive_expect_tx(bar_load, 2 * kStTile);
    for (int half = 0; half < 2; ++half) {
      tma_load_4d(sA + half * kStBox, &tmA, bar_load, half * 64, 0, 0, 0);
      tma_load_4d(sB + half * kStBox, &tmB, bar_load, half * 64, 0, 0, 0);
    }
  }
  mbar_wait(bar_load, 0);

  if (mode == 2) {
    const uint16_t* s16 = reinterpret_cast<const uint16_t*>(sA);
    uint16_t* o16 = static_cast<uint16_t*>(out);
    for (int i = t; i < kStBox / 2; i += 128) o16[i] = s16[i];
    return;
  }
  const uint32_t a0 = smem_u32(sA), b0 = smem_u32(sB);
  for (int hm = 0; hm < 2; ++hm) {
    float d[64];
    wgmma_fence();
    if (mode == 0) {
      for (int kk = 0; kk < 8; ++kk) {
        const uint32_t off = (kk >> 2) * kStBox + (kk & 3) * 32;
        wgmma_ss_n128<kBF16, 0, 0>(d, make_desc(a0 + hm * 64 * 128 + off, 16, 1024), make_desc(b0 + off, 16, 1024),
                                   kk > 0 ? 1u : 0u);
      }
    } else if (mode == 1) {
      // A fragment straight from global memory: row 64 hm + 16 w + g (+ 8), columns 16 kk + 2 q (+ 8)
      const uint32_t* src = reinterpret_cast<const uint32_t*>(a_raw);
      const int row = 64 * hm + 16 * w + g;
      for (int kk = 0; kk < 8; ++kk) {
        uint32_t a[4];
        a[0] = src[(row * 128 + 16 * kk + 2 * q) / 2];
        a[1] = src[((row + 8) * 128 + 16 * kk + 2 * q) / 2];
        a[2] = src[(row * 128 + 16 * kk + 8 + 2 * q) / 2];
        a[3] = src[((row + 8) * 128 + 16 * kk + 8 + 2 * q) / 2];
        fence_regs<4>(a);
        wgmma_rs_n128<kBF16, 1>(d, a, make_desc(b0 + kk * 2048, kStBox, 1024), kk > 0 ? 1u : 0u);
      }
    } else {  // mode 3: both operands MN-major: A stored [k][m], B stored [k][n]
      for (int kk = 0; kk < 8; ++kk)
        wgmma_ss_n128<kBF16, 1, 1>(d, make_desc(a0 + hm * kStBox + kk * 2048, kStBox, 1024),
                                   make_desc(b0 + kk * 2048, kStBox, 1024), kk > 0 ? 1u : 0u);
    }
    wgmma_commit();
    wgmma_wait<0>();
    fence_regs<64>(d);
    float* o = static_cast<float*>(out);
    for (int c = 0; c < 16; ++c)
      for (int r = 0; r < 2; ++r) {
        const int row = 64 * hm + 16 * w + g + 8 * r;
        o[row * 128 + 8 * c + 2 * q] = d[4 * c + 2 * r];
        o[row * 128 + 8 * c + 2 * q + 1] = d[4 * c + 2 * r + 1];
      }
  }
}

}  // namespace ba

extern "C" int ba_selftest(int mode, const void* a, const void* b, void* out, int dtype, void* stream) {
  using namespace ba;
  BA_REQUIRE(mode >= 0 && mode <= 3, "ba_selftest: bad mode %d", mode);
  BA_REQUIRE(a && b && out, "ba_selftest: null pointer");
  ba_tensor4 ta{const_cast<void*>(a), 128 * 128, 128, 128};
  ba_tensor4 tb{const_cast<void*>(b), 128 * 128, 128, 128};
  CUtensorMap tmA, tmB;
  int rc;
  if ((rc = make_tensor_map(&tmA, ta, 1, 128, 1, 128, lowp_dtype(dtype), 2, 64, 128, true))) return rc;
  if ((rc = make_tensor_map(&tmB, tb, 1, 128, 1, 128, lowp_dtype(dtype), 2, 64, 128, true))) return rc;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (dtype == BA_DTYPE_BF16) {
    BA_CHECK_CUDA(cudaFuncSetAttribute(selftest_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, kStSmem));
    selftest_kernel<true><<<1, 128, kStSmem, st>>>(tmA, tmB, static_cast<const uint16_t*>(a), out, mode);
  } else {
    BA_CHECK_CUDA(cudaFuncSetAttribute(selftest_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, kStSmem));
    selftest_kernel<false><<<1, 128, kStSmem, st>>>(tmA, tmB, static_cast<const uint16_t*>(a), out, mode);
  }
  BA_CHECK_CUDA(cudaGetLastError());
  return BA_OK;
}
