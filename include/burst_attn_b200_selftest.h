/* burst_attn_b200_selftest -- diagnostics of the sm_90a building blocks.  NOT part of the drop-in boundary:
 * these entry points live in their own library (libburst_attn_b200_selftest.so) that only tests/ and tools/ load.
 * Same conventions as burst_attn_b200.h (status codes, ba_last_error of the main library is not shared: this
 * library exports ba_selftest_last_error).                                                                   */
#ifndef BURST_ATTN_B200_SELFTEST_H
#define BURST_ATTN_B200_SELFTEST_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

const char* ba_selftest_last_error(void);

/* ---- self tests of the sm_90a building blocks (tests/ only) --------------------
 * mode 0: S[128,128] fp32 = A[128,128] * B[128,128]^T through TMA + wgmma SS (both operands K-major)
 * mode 1: O[128,128] fp32 = P[128,128] * V[128,128] with P in registers (wgmma RS, V MN-major)
 * mode 2: raw dump of a TMA-loaded 128x64 SWIZZLE_128B box (16 KiB)
 * mode 3: out = A^T * B with both operands MN-major (backward's dQ path)
 * a, b: dtype [128,128] row-major; out: fp32 [128,128] (mode 2: 8192 x 16-bit).                               */
int ba_selftest(int mode, const void* a, const void* b, void* out, int dtype, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* BURST_ATTN_B200_SELFTEST_H */
