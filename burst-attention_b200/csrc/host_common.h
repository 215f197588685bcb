// Host-side helpers shared by the C-ABI entry points: thread-local error string,
// CUDA error mapping, argument checks, and TMA tensor-map construction through
// the driver entry point (no link-time dependency on libcuda).
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdarg.h>
#include <stdint.h>
#include <stdio.h>

#include "burst_attn_b200.h"

namespace ba {

void set_error(const char* fmt, ...);
int cuda_fail(cudaError_t e, const char* what);

#define BA_CHECK_CUDA(expr)                                  \
  do {                                                       \
    cudaError_t _e = (expr);                                 \
    if (_e != cudaSuccess) return ::ba::cuda_fail(_e, #expr); \
  } while (0)

#define BA_REQUIRE(cond, ...)          \
  do {                                 \
    if (!(cond)) {                     \
      ::ba::set_error(__VA_ARGS__);    \
      return BA_ERR_INVALID;           \
    }                                  \
  } while (0)

// Build a 4-D tiled tensor map over a [b,s,h,d] view (d contiguous):
// dims innermost-first (D, H, S, B); box (box_d, 1, box_s, 1).
// esize: element size in bytes; swizzle128: CU_TENSOR_MAP_SWIZZLE_128B when
// box_d*esize == 128, else no swizzle.
int make_tensor_map(CUtensorMap* out, const ba_tensor4& t, int B, int S, int H, int D, CUtensorMapDataType dt,
                    int esize, int box_d, int box_s, bool swizzle128);

inline CUtensorMapDataType lowp_dtype(int dtype) {
  return dtype == BA_DTYPE_BF16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16;
}

// A view the kernels can access with 16-byte loads and stores: 16-byte aligned base, every stride a multiple of
// 16 bytes (esize: element size in bytes).  A null pointer passes; callers that need one check for it.
inline bool aligned16(const ba_tensor4& t, int esize) {
  const int q = 16 / esize;
  return (reinterpret_cast<uintptr_t>(t.ptr) & 15) == 0 && t.stride_b % q == 0 && t.stride_s % q == 0 &&
         t.stride_h % q == 0;
}

// The arguments of one forward or backward chunk call besides its operands: the problem, the mask, and the optional
// key bias, ALiBi and documents.  Fields up to lower_offset are in the entry points' parameter order.
struct ChunkArgs {
  int B, Sq, Sk, H, H_kv, D;
  float scale;
  int mask_mode, causal_offset, lower_offset;
  int dtype;
  ba_rowstat key_bias = {nullptr, 0, 0};  // null: no key bias
  const float* slopes = nullptr;          // ALiBi; null: none
  int64_t slopes_stride_b = 0, dist0 = 0;
  const int* cu_seqlens = nullptr;        // documents; null: none
  int n_docs = 0;
  int64_t q_pos0 = 0, k_pos0 = 0;
  int pstride = 1;                        // ALiBi and documents
};

// Which family of entry points a chunk call came through, and so which of its arguments are checked.
//   kPlain  ba_*_chunk, _bias, _gqa: mask_mode is BA_MASK_NONE or BA_MASK_CAUSAL
//   kBand   ba_*_chunk_band: mask_mode is a set of BA_MASK_CAUSAL and BA_MASK_LOWER bits
//   kAlibi  ba_*_chunk_alibi: the band's masks, plus the slopes (non-null, 4-byte aligned, batch stride >= 0) and
//           pstride >= 1
//   kDoc    ba_*_chunk_doc: the band's masks, plus the boundaries (non-null, 4-byte aligned, n_docs >= 1),
//           pstride >= 1 and positions q_pos0, k_pos0 >= 0 whose last row and key still fit in int32
enum class ChunkEntry { kPlain, kBand, kAlibi, kDoc };

// The preconditions of every forward and backward chunk entry point; `fn` names the entry point in the error message.
// Returns BA_OK or BA_ERR_INVALID.  On success it normalises the masks without changing which keys are visible:
// causal_offset is clamped into [-Sq, Sk] (beyond either end it shows every key or none, and the kernels' 32-bit index
// sums with it stay in range), a lower edge that masks nothing is dropped from mask_mode, and lower_offset is clamped
// to Sk -- still at or below the clamped causal offset.  Documents always run with a lower edge: without
// BA_MASK_LOWER it is 1 - Sq, which masks nothing.
int check_chunk_args(const char* fn, ChunkEntry entry, ChunkArgs* a);

}  // namespace ba
