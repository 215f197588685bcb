#include "host_common.h"

#include <math.h>
#include <mutex>
#include <string.h>

namespace ba {

static thread_local char g_err[512] = "";

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

int cuda_fail(cudaError_t e, const char* what) {
  set_error("CUDA error %d (%s) at %s", static_cast<int>(e), cudaGetErrorString(e), what);
  return BA_ERR_CUDA;
}

typedef CUresult (*encode_tiled_fn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static encode_tiled_fn get_encode() {
  static encode_tiled_fn fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess) {
      fn = reinterpret_cast<encode_tiled_fn>(p);
    }
  });
  return fn;
}

int make_tensor_map(CUtensorMap* out, const ba_tensor4& t, int B, int S, int H, int D, CUtensorMapDataType dt,
                    int esize, int box_d, int box_s, bool swizzle128) {
  encode_tiled_fn enc = get_encode();
  if (!enc) {
    set_error("cuTensorMapEncodeTiled driver entry point not available");
    return BA_ERR_CUDA;
  }
  if ((reinterpret_cast<uintptr_t>(t.ptr) & 15) != 0) {
    set_error("tensor base pointer must be 16-byte aligned for TMA");
    return BA_ERR_INVALID;
  }
  // A dimension of extent 1 never contributes to an address; give it a legal stride.
  int64_t sh = (H == 1) ? D : t.stride_h;
  int64_t ss = (S == 1) ? (int64_t)D * H : t.stride_s;
  int64_t sb = (B == 1) ? ss * S : t.stride_b;
  if (B == 1 && sb < (int64_t)D) sb = (int64_t)D * H * S;
  cuuint64_t dims[4] = {(cuuint64_t)D, (cuuint64_t)H, (cuuint64_t)S, (cuuint64_t)B};
  cuuint64_t strides[3] = {(cuuint64_t)sh * esize, (cuuint64_t)ss * esize, (cuuint64_t)sb * esize};
  for (int i = 0; i < 3; ++i) {
    if (strides[i] % 16 != 0 || strides[i] == 0) {
      set_error("tensor stride %d (= %llu bytes) must be a positive multiple of 16 bytes for TMA", i,
                (unsigned long long)strides[i]);
      return BA_ERR_INVALID;
    }
  }
  cuuint32_t box[4] = {(cuuint32_t)box_d, 1u, (cuuint32_t)box_s, 1u};
  cuuint32_t estr[4] = {1u, 1u, 1u, 1u};
  CUresult r = enc(out, dt, 4, t.ptr, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                   swizzle128 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_NONE,
                   CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled failed with CUresult %d (dims %d,%d,%d,%d box %d,%d)", (int)r, D, H, S, B,
              box_d, box_s);
    return BA_ERR_CUDA;
  }
  return BA_OK;
}

int check_chunk_args(const char* fn, int B, int Sq, int Sk, int H, int H_kv, int D, float scale, int mask_mode,
                     int dtype) {
  BA_REQUIRE(H_kv > 0 && H % H_kv == 0, "%s: H_kv=%d must be positive and divide H=%d", fn, H_kv, H);
  BA_REQUIRE(D == 128 || D == 64, "%s: head dim %d unsupported (64 or 128)", fn, D);
  BA_REQUIRE(B > 0 && Sq > 0 && Sk > 0 && H > 0, "%s: empty problem B=%d Sq=%d Sk=%d H=%d", fn, B, Sq, Sk, H);
  BA_REQUIRE(dtype == BA_DTYPE_FP16 || dtype == BA_DTYPE_BF16, "%s: bad dtype %d", fn, dtype);
  BA_REQUIRE(mask_mode == BA_MASK_NONE || mask_mode == BA_MASK_CAUSAL, "%s: bad mask mode %d", fn, mask_mode);
  BA_REQUIRE(scale > 0.f && isfinite(scale), "%s: softmax scale must be positive and finite", fn);
  BA_REQUIRE(H <= 65535 && B <= 65535, "%s: H and B must be <= 65535", fn);  // gridDim.y / gridDim.z
  return BA_OK;
}

int check_band_args(const char* fn, int B, int Sq, int Sk, int H, int H_kv, int D, float scale, int* mask_mode,
                    int* causal_offset, int* lower_offset, int dtype) {
  const int mm = *mask_mode;
  BA_REQUIRE((mm & ~(BA_MASK_CAUSAL | BA_MASK_LOWER)) == 0, "%s: bad mask mode %d", fn, mm);
  int rc;
  if ((rc = check_chunk_args(fn, B, Sq, Sk, H, H_kv, D, scale, mm & BA_MASK_CAUSAL, dtype))) return rc;
  BA_REQUIRE(!(mm & BA_MASK_LOWER) || !(mm & BA_MASK_CAUSAL) || *lower_offset <= *causal_offset,
             "%s: band lower_offset %d is above its causal_offset %d (no key would be visible)", fn, *lower_offset,
             *causal_offset);
  // The kernels add the causal offset to row and key indices in 32-bit arithmetic.  An offset >= Sk - 1 shows every
  // key to every row and one <= -Sq shows none, so clamping it into [-Sq, Sk] changes no mask and keeps those sums in
  // range.  A lower edge at or below the causal one stays there: both clamps below are monotone, and a clamped lower
  // edge is at most Sk.
  *causal_offset = *causal_offset > Sk ? Sk : *causal_offset < -Sq ? -Sq : *causal_offset;
  if (!(mm & BA_MASK_LOWER)) return BA_OK;
  // a lower edge at or below key 0 for every row (lower_offset <= 1 - Sq) masks nothing: run the kernel without one;
  // one at or above Sk masks every key of every row, as lower_offset = Sk does (and row + Sk cannot overflow)
  if (*lower_offset <= 1 - Sq) *mask_mode = mm & ~BA_MASK_LOWER;
  else if (*lower_offset > Sk) *lower_offset = Sk;
  return BA_OK;
}

int check_alibi_args(const char* fn, int B, int Sq, int Sk, int H, int H_kv, int D, float scale, int* mask_mode,
                     int* causal_offset, int* lower_offset, const float* slopes, int64_t slopes_stride_b, int pstride,
                     int dtype) {
  int rc;
  if ((rc = check_band_args(fn, B, Sq, Sk, H, H_kv, D, scale, mask_mode, causal_offset, lower_offset, dtype)))
    return rc;
  BA_REQUIRE(slopes, "%s: null ALiBi slopes", fn);
  BA_REQUIRE((reinterpret_cast<uintptr_t>(slopes) & 3) == 0, "%s: ALiBi slopes must be 4-byte aligned", fn);
  BA_REQUIRE(slopes_stride_b >= 0, "%s: ALiBi slopes batch stride %lld is negative", fn, (long long)slopes_stride_b);
  BA_REQUIRE(pstride >= 1, "%s: ALiBi position stride %d must be >= 1", fn, pstride);
  return BA_OK;
}

int check_doc_args(const char* fn, int B, int Sq, int Sk, int H, int H_kv, int D, float scale, int* mask_mode,
                   int* causal_offset, int* lower_offset, const int* cu_seqlens, int n_docs, int64_t q_pos0,
                   int64_t k_pos0, int pstride, int dtype) {
  int rc;
  if ((rc = check_band_args(fn, B, Sq, Sk, H, H_kv, D, scale, mask_mode, causal_offset, lower_offset, dtype)))
    return rc;
  BA_REQUIRE(cu_seqlens, "%s: null cu_seqlens", fn);
  BA_REQUIRE((reinterpret_cast<uintptr_t>(cu_seqlens) & 3) == 0, "%s: cu_seqlens must be 4-byte aligned", fn);
  BA_REQUIRE(n_docs >= 1, "%s: n_docs = %d must be >= 1", fn, n_docs);
  BA_REQUIRE(pstride >= 1, "%s: position stride %d must be >= 1", fn, pstride);
  BA_REQUIRE(q_pos0 >= 0 && k_pos0 >= 0, "%s: positions q_pos0 = %lld, k_pos0 = %lld must be >= 0", fn,
             (long long)q_pos0, (long long)k_pos0);
  // cu_seqlens is int32, so every position is; the kernels count positions in 32 bits
  BA_REQUIRE(q_pos0 + (int64_t)pstride * (Sq - 1) <= INT32_MAX && k_pos0 + (int64_t)pstride * (Sk - 1) <= INT32_MAX,
             "%s: the positions of the rows or keys exceed int32", fn);
  return BA_OK;
}

}  // namespace ba

#ifdef BA_SELFTEST_LIB
extern "C" const char* ba_selftest_last_error(void) { return ba::g_err; }
#else
extern "C" const char* ba_last_error(void) { return ba::g_err; }
// 201: grouped-query attention (ba_fwd_chunk_gqa, ba_bwd_chunk_gqa); 202: band masks (ba_fwd_chunk_band,
// ba_bwd_chunk_band)
// 203: ALiBi (ba_fwd_chunk_alibi, ba_bwd_chunk_alibi)
// 204: packed documents (ba_fwd_chunk_doc, ba_bwd_chunk_doc)
extern "C" int ba_version(void) { return 204; }
extern "C" int ba_device_check(void) {
  int dev = 0;
  BA_CHECK_CUDA(cudaGetDevice(&dev));
  int major = 0, minor = 0;
  BA_CHECK_CUDA(cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev));
  BA_CHECK_CUDA(cudaDeviceGetAttribute(&minor, cudaDevAttrComputeCapabilityMinor, dev));
  if (major != 9 || minor != 0) {
    ba::set_error("burst_attn_b200 needs an sm_90 (H100) device, found sm_%d%d", major, minor);
    return BA_ERR_UNSUPPORTED;
  }
  return BA_OK;
}
#endif
