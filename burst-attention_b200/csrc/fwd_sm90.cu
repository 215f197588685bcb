// ba_fwd_chunk*: the forward entry points, and the tile kernel without a band's lower edge (fwd_sm90.cuh).
#include "fwd_sm90.cuh"

namespace ba {

// Every forward entry point after its argument check: fill FwdParams and launch the tile kernel of the call's masks.
static int fwd_chunk_run(ba_tensor4 q, ba_tensor4 k, ba_tensor4 v, ba_tensor4 o_acc, ba_rowstat lse,
                         ba_tensor4 o_out, const ChunkArgs& a, int flags, void* stream) {
  int rc;
  BA_REQUIRE(q.ptr && k.ptr && v.ptr && lse.ptr, "ba_fwd_chunk: null q/k/v/lse");
  const bool first = flags & BA_FWD_FIRST, last = flags & BA_FWD_LAST;
  BA_REQUIRE(!last || o_out.ptr, "ba_fwd_chunk: BA_FWD_LAST needs o_out");
  BA_REQUIRE((first && last) || o_acc.ptr, "ba_fwd_chunk: fp32 state o_acc required unless FIRST|LAST");
  if (o_acc.ptr)
    BA_REQUIRE(aligned16(o_acc, 4), "ba_fwd_chunk: o_acc must be 16-byte aligned with strides multiple of 4 elements");
  if (o_out.ptr)
    BA_REQUIRE(aligned16(o_out, 2), "ba_fwd_chunk: o_out must be 16-byte aligned with strides multiple of 8 elements");

  CUtensorMap tmQ, tmK, tmV;
  const CUtensorMapDataType dt = lowp_dtype(a.dtype);
  if ((rc = make_tensor_map(&tmQ, q, a.B, a.Sq, a.H, a.D, dt, 2, 64, kBlockM, true))) return rc;
  if ((rc = make_tensor_map(&tmK, k, a.B, a.Sk, a.H_kv, a.D, dt, 2, 64, kBlockN, true))) return rc;
  if ((rc = make_tensor_map(&tmV, v, a.B, a.Sk, a.H_kv, a.D, dt, 2, 64, kBlockN, true))) return rc;

  FwdParams p;
  p.o_acc = static_cast<float*>(o_acc.ptr);
  p.oacc_sb = o_acc.stride_b, p.oacc_ss = o_acc.stride_s, p.oacc_sh = o_acc.stride_h;
  p.lse = lse.ptr;
  p.lse_sb = lse.stride_b, p.lse_sh = lse.stride_h;
  p.o_out = o_out.ptr;
  p.oout_sb = o_out.stride_b, p.oout_ss = o_out.stride_s, p.oout_sh = o_out.stride_h;
  p.B = a.B, p.Sq = a.Sq, p.Sk = a.Sk, p.H = a.H;
  p.G = a.H / a.H_kv;
  p.scale_log2 = a.scale * kLog2e;
  p.causal = (a.mask_mode & BA_MASK_CAUSAL) != 0;
  p.causal_off = a.causal_offset;
  p.load_state = first ? 0 : 1;
  p.store_lowp = last ? 1 : 0;
  p.lo = a.lower_offset;
  p.bias = a.key_bias.ptr, p.bias_sb = a.key_bias.stride_b, p.bias_sh = a.key_bias.stride_h;
  p.slopes = a.slopes, p.slopes_sb = a.slopes_stride_b, p.dist0 = a.dist0, p.pstride = a.pstride;
  p.cu = a.cu_seqlens, p.n_docs = a.n_docs, p.q_pos0 = (int)a.q_pos0, p.k_pos0 = (int)a.k_pos0;  // checked: they fit

  const bool bf16 = a.dtype == BA_DTYPE_BF16, lower = a.mask_mode & BA_MASK_LOWER, bias = a.key_bias.ptr;
  const FwdKernel kern = a.cu_seqlens ? fwd_doc_kernel_of(bf16, a.D)
                         : a.slopes   ? fwd_alibi_kernel_of(bf16, a.D, lower)
                         : lower      ? fwd_band_kernel_of(bf16, a.D, bias)
                                      : fwd_chunk_kernel_of<false>(bf16, a.D, bias);
  const int smem = a.D == 64 ? FwdLayout<64>::kSmemBytes : FwdLayout<128>::kSmemBytes;
  BA_CHECK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  dim3 grid((a.Sq + kBlockM - 1) / kBlockM, a.H, a.B);
  kern<<<grid, kFwdThreads, smem, static_cast<cudaStream_t>(stream)>>>(tmQ, tmK, tmV, p);
  BA_CHECK_CUDA(cudaGetLastError());
  return BA_OK;
}

}  // namespace ba

extern "C" int ba_fwd_chunk(ba_tensor4 q, ba_tensor4 k, ba_tensor4 v, ba_tensor4 o_acc, ba_rowstat lse,
                            ba_tensor4 o_out, int B, int Sq, int Sk, int H, int D, float scale, int mask_mode,
                            int causal_offset, int flags, int dtype, void* stream) {
  ba_rowstat none = {nullptr, 0, 0};
  return ba_fwd_chunk_bias(q, k, v, none, o_acc, lse, o_out, B, Sq, Sk, H, D, scale, mask_mode, causal_offset, flags,
                           dtype, stream);
}

extern "C" int ba_fwd_chunk_bias(ba_tensor4 q, ba_tensor4 k, ba_tensor4 v, ba_rowstat key_bias, ba_tensor4 o_acc,
                                 ba_rowstat lse, ba_tensor4 o_out, int B, int Sq, int Sk, int H, int D, float scale,
                                 int mask_mode, int causal_offset, int flags, int dtype, void* stream) {
  return ba_fwd_chunk_gqa(q, k, v, key_bias, o_acc, lse, o_out, B, Sq, Sk, H, H, D, scale, mask_mode, causal_offset,
                          flags, dtype, stream);
}

extern "C" int ba_fwd_chunk_gqa(ba_tensor4 q, ba_tensor4 k, ba_tensor4 v, ba_rowstat key_bias, ba_tensor4 o_acc,
                                ba_rowstat lse, ba_tensor4 o_out, int B, int Sq, int Sk, int H, int H_kv, int D,
                                float scale, int mask_mode, int causal_offset, int flags, int dtype, void* stream) {
  ba::ChunkArgs a{B, Sq, Sk, H, H_kv, D, scale, mask_mode, causal_offset, 0, dtype};
  a.key_bias = key_bias;
  const int rc = ba::check_chunk_args("ba_fwd_chunk", ba::ChunkEntry::kPlain, &a);
  return rc ? rc : ba::fwd_chunk_run(q, k, v, o_acc, lse, o_out, a, flags, stream);
}

extern "C" int ba_fwd_chunk_band(ba_tensor4 q, ba_tensor4 k, ba_tensor4 v, ba_rowstat key_bias, ba_tensor4 o_acc,
                                 ba_rowstat lse, ba_tensor4 o_out, int B, int Sq, int Sk, int H, int H_kv, int D,
                                 float scale, int mask_mode, int causal_offset, int lower_offset, int flags, int dtype,
                                 void* stream) {
  ba::ChunkArgs a{B, Sq, Sk, H, H_kv, D, scale, mask_mode, causal_offset, lower_offset, dtype};
  a.key_bias = key_bias;
  const int rc = ba::check_chunk_args("ba_fwd_chunk", ba::ChunkEntry::kBand, &a);
  return rc ? rc : ba::fwd_chunk_run(q, k, v, o_acc, lse, o_out, a, flags, stream);
}

extern "C" int ba_fwd_chunk_alibi(ba_tensor4 q, ba_tensor4 k, ba_tensor4 v, ba_tensor4 o_acc, ba_rowstat lse,
                                  ba_tensor4 o_out, int B, int Sq, int Sk, int H, int H_kv, int D, float scale,
                                  int mask_mode, int causal_offset, int lower_offset, const float* slopes,
                                  int64_t slopes_stride_b, int64_t dist0, int pstride, int flags, int dtype,
                                  void* stream) {
  ba::ChunkArgs a{B, Sq, Sk, H, H_kv, D, scale, mask_mode, causal_offset, lower_offset, dtype};
  a.slopes = slopes, a.slopes_stride_b = slopes_stride_b, a.dist0 = dist0, a.pstride = pstride;
  const int rc = ba::check_chunk_args("ba_fwd_chunk_alibi", ba::ChunkEntry::kAlibi, &a);
  return rc ? rc : ba::fwd_chunk_run(q, k, v, o_acc, lse, o_out, a, flags, stream);
}

extern "C" int ba_fwd_chunk_doc(ba_tensor4 q, ba_tensor4 k, ba_tensor4 v, ba_tensor4 o_acc, ba_rowstat lse,
                                ba_tensor4 o_out, int B, int Sq, int Sk, int H, int H_kv, int D, float scale,
                                int mask_mode, int causal_offset, int lower_offset, const int* cu_seqlens, int n_docs,
                                int64_t q_pos0, int64_t k_pos0, int pstride, int flags, int dtype, void* stream) {
  ba::ChunkArgs a{B, Sq, Sk, H, H_kv, D, scale, mask_mode, causal_offset, lower_offset, dtype};
  a.cu_seqlens = cu_seqlens, a.n_docs = n_docs, a.q_pos0 = q_pos0, a.k_pos0 = k_pos0, a.pstride = pstride;
  const int rc = ba::check_chunk_args("ba_fwd_chunk_doc", ba::ChunkEntry::kDoc, &a);
  return rc ? rc : ba::fwd_chunk_run(q, k, v, o_acc, lse, o_out, a, flags, stream);
}
