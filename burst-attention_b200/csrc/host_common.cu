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

int check_chunk_args(const char* fn, ChunkEntry entry, ChunkArgs* a) {
  const int mm = a->mask_mode;
  const int masks = entry == ChunkEntry::kPlain ? BA_MASK_CAUSAL : BA_MASK_CAUSAL | BA_MASK_LOWER;
  // the band's entry points report a bad mask mode before anything else, the plain ones after the dtype
  if (entry != ChunkEntry::kPlain) BA_REQUIRE((mm & ~masks) == 0, "%s: bad mask mode %d", fn, mm);
  BA_REQUIRE(a->H_kv > 0 && a->H % a->H_kv == 0, "%s: H_kv=%d must be positive and divide H=%d", fn, a->H_kv, a->H);
  BA_REQUIRE(a->D == 128 || a->D == 64, "%s: head dim %d unsupported (64 or 128)", fn, a->D);
  BA_REQUIRE(a->B > 0 && a->Sq > 0 && a->Sk > 0 && a->H > 0, "%s: empty problem B=%d Sq=%d Sk=%d H=%d", fn, a->B,
             a->Sq, a->Sk, a->H);
  BA_REQUIRE(a->dtype == BA_DTYPE_FP16 || a->dtype == BA_DTYPE_BF16, "%s: bad dtype %d", fn, a->dtype);
  BA_REQUIRE((mm & ~masks) == 0, "%s: bad mask mode %d", fn, mm);
  BA_REQUIRE(a->scale > 0.f && isfinite(a->scale), "%s: softmax scale must be positive and finite", fn);
  BA_REQUIRE(a->H <= 65535 && a->B <= 65535, "%s: H and B must be <= 65535", fn);  // gridDim.y / gridDim.z
  BA_REQUIRE(!(mm & BA_MASK_LOWER) || !(mm & BA_MASK_CAUSAL) || a->lower_offset <= a->causal_offset,
             "%s: band lower_offset %d is above its causal_offset %d (no key would be visible)", fn, a->lower_offset,
             a->causal_offset);
  if (entry == ChunkEntry::kAlibi) {
    BA_REQUIRE(a->slopes, "%s: null ALiBi slopes", fn);
    BA_REQUIRE((reinterpret_cast<uintptr_t>(a->slopes) & 3) == 0, "%s: ALiBi slopes must be 4-byte aligned", fn);
    BA_REQUIRE(a->slopes_stride_b >= 0, "%s: ALiBi slopes batch stride %lld is negative", fn,
               (long long)a->slopes_stride_b);
    BA_REQUIRE(a->pstride >= 1, "%s: ALiBi position stride %d must be >= 1", fn, a->pstride);
  }
  if (entry == ChunkEntry::kDoc) {
    BA_REQUIRE(a->cu_seqlens, "%s: null cu_seqlens", fn);
    BA_REQUIRE((reinterpret_cast<uintptr_t>(a->cu_seqlens) & 3) == 0, "%s: cu_seqlens must be 4-byte aligned", fn);
    BA_REQUIRE(a->n_docs >= 1, "%s: n_docs = %d must be >= 1", fn, a->n_docs);
    BA_REQUIRE(a->pstride >= 1, "%s: position stride %d must be >= 1", fn, a->pstride);
    BA_REQUIRE(a->q_pos0 >= 0 && a->k_pos0 >= 0, "%s: positions q_pos0 = %lld, k_pos0 = %lld must be >= 0", fn,
               (long long)a->q_pos0, (long long)a->k_pos0);
    // cu_seqlens is int32, so every position is; the kernels count positions in 32 bits
    BA_REQUIRE(a->q_pos0 + (int64_t)a->pstride * (a->Sq - 1) <= INT32_MAX &&
                   a->k_pos0 + (int64_t)a->pstride * (a->Sk - 1) <= INT32_MAX,
               "%s: the positions of the rows or keys exceed int32", fn);
  }
  // The kernels add the causal offset to row and key indices in 32-bit arithmetic.  An offset >= Sk - 1 shows every
  // key to every row and one <= -Sq shows none, so clamping it into [-Sq, Sk] changes no mask and keeps those sums in
  // range.  A lower edge at or below the causal one stays there: both clamps below are monotone, and a clamped lower
  // edge is at most Sk.
  a->causal_offset = a->causal_offset > a->Sk ? a->Sk : a->causal_offset < -a->Sq ? -a->Sq : a->causal_offset;
  // a lower edge at or below key 0 for every row (lower_offset <= 1 - Sq) masks nothing: run the kernel without one;
  // one at or above Sk masks every key of every row, as lower_offset = Sk does (and row + Sk cannot overflow)
  if (mm & BA_MASK_LOWER) {
    if (a->lower_offset <= 1 - a->Sq) a->mask_mode = mm & ~BA_MASK_LOWER;
    else if (a->lower_offset > a->Sk) a->lower_offset = a->Sk;
  }
  // documents run on the band path: without a lower edge, one that masks nothing (row + 1 - Sq <= 0 <= key)
  if (entry == ChunkEntry::kDoc && !(a->mask_mode & BA_MASK_LOWER)) a->lower_offset = 1 - a->Sq;
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
