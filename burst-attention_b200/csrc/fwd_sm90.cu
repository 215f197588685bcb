// ba_fwd_chunk*: the forward entry points, and the tile kernel without a band's lower edge (fwd_sm90.cuh).
#include "fwd_sm90.cuh"

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
  int rc;  // no band here: only BA_MASK_NONE / BA_MASK_CAUSAL
  if ((rc = ba::check_chunk_args("ba_fwd_chunk", B, Sq, Sk, H, H_kv, D, scale, mask_mode, dtype))) return rc;
  return ba_fwd_chunk_band(q, k, v, key_bias, o_acc, lse, o_out, B, Sq, Sk, H, H_kv, D, scale, mask_mode,
                           causal_offset, 0, flags, dtype, stream);
}

namespace ba {

// ba_fwd_chunk_band, ba_fwd_chunk_alibi and ba_fwd_chunk_doc after their argument checks (slopes: ALiBi, else null;
// cu: documents, else null)
static int fwd_chunk_run(ba_tensor4 q, ba_tensor4 k, ba_tensor4 v, ba_rowstat key_bias, ba_tensor4 o_acc,
                         ba_rowstat lse, ba_tensor4 o_out, int B, int Sq, int Sk, int H, int H_kv, int D, float scale,
                         int mask_mode, int causal_offset, int lower_offset, const float* slopes,
                         int64_t slopes_stride_b, int64_t dist0, int pstride, const int* cu, int n_docs,
                         int64_t q_pos0, int64_t k_pos0, int flags, int dtype, void* stream) {
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
  const CUtensorMapDataType dt = lowp_dtype(dtype);
  if ((rc = make_tensor_map(&tmQ, q, B, Sq, H, D, dt, 2, 64, kBlockM, true))) return rc;
  if ((rc = make_tensor_map(&tmK, k, B, Sk, H_kv, D, dt, 2, 64, kBlockN, true))) return rc;
  if ((rc = make_tensor_map(&tmV, v, B, Sk, H_kv, D, dt, 2, 64, kBlockN, true))) return rc;

  FwdParams p;
  p.o_acc = static_cast<float*>(o_acc.ptr);
  p.oacc_sb = o_acc.stride_b, p.oacc_ss = o_acc.stride_s, p.oacc_sh = o_acc.stride_h;
  p.lse = lse.ptr;
  p.lse_sb = lse.stride_b, p.lse_sh = lse.stride_h;
  p.o_out = o_out.ptr;
  p.oout_sb = o_out.stride_b, p.oout_ss = o_out.stride_s, p.oout_sh = o_out.stride_h;
  p.B = B, p.Sq = Sq, p.Sk = Sk, p.H = H;
  p.G = H / H_kv;
  p.scale_log2 = scale * kLog2e;
  p.causal = (mask_mode & BA_MASK_CAUSAL) != 0;
  p.causal_off = causal_offset;
  p.load_state = first ? 0 : 1;
  p.store_lowp = last ? 1 : 0;
  p.lo = lower_offset;
  p.bias = key_bias.ptr, p.bias_sb = key_bias.stride_b, p.bias_sh = key_bias.stride_h;
  p.slopes = slopes, p.slopes_sb = slopes_stride_b, p.dist0 = dist0, p.pstride = pstride;
  p.cu = cu, p.n_docs = n_docs, p.q_pos0 = (int)q_pos0, p.k_pos0 = (int)k_pos0;  // check_doc_args: they fit
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  const bool bias = key_bias.ptr != nullptr;
  if (cu) {  // the band path, with a lower edge that masks nothing when there is none (row + 1 - Sq <= 0 <= key)
    if (!(mask_mode & BA_MASK_LOWER)) p.lo = 1 - Sq;
    return launch_fwd_doc(dtype, D, tmQ, tmK, tmV, p, st);
  }
  if (slopes) return launch_fwd_alibi(dtype, D, (mask_mode & BA_MASK_LOWER) != 0, tmQ, tmK, tmV, p, st);
  if (mask_mode & BA_MASK_LOWER) return launch_fwd_band(dtype, D, bias, tmQ, tmK, tmV, p, st);
  return launch_fwd<false>(dtype, D, bias, tmQ, tmK, tmV, p, st);
}

}  // namespace ba

extern "C" int ba_fwd_chunk_band(ba_tensor4 q, ba_tensor4 k, ba_tensor4 v, ba_rowstat key_bias, ba_tensor4 o_acc,
                                 ba_rowstat lse, ba_tensor4 o_out, int B, int Sq, int Sk, int H, int H_kv, int D,
                                 float scale, int mask_mode, int causal_offset, int lower_offset, int flags, int dtype,
                                 void* stream) {
  int rc;
  if ((rc = ba::check_band_args("ba_fwd_chunk", B, Sq, Sk, H, H_kv, D, scale, &mask_mode, &causal_offset,
                                &lower_offset, dtype)))
    return rc;
  return ba::fwd_chunk_run(q, k, v, key_bias, o_acc, lse, o_out, B, Sq, Sk, H, H_kv, D, scale, mask_mode,
                           causal_offset, lower_offset, nullptr, 0, 0, 1, nullptr, 0, 0, 0, flags, dtype, stream);
}

extern "C" int ba_fwd_chunk_alibi(ba_tensor4 q, ba_tensor4 k, ba_tensor4 v, ba_tensor4 o_acc, ba_rowstat lse,
                                  ba_tensor4 o_out, int B, int Sq, int Sk, int H, int H_kv, int D, float scale,
                                  int mask_mode, int causal_offset, int lower_offset, const float* slopes,
                                  int64_t slopes_stride_b, int64_t dist0, int pstride, int flags, int dtype,
                                  void* stream) {
  int rc;
  if ((rc = ba::check_alibi_args("ba_fwd_chunk_alibi", B, Sq, Sk, H, H_kv, D, scale, &mask_mode, &causal_offset,
                                 &lower_offset, slopes, slopes_stride_b, pstride, dtype)))
    return rc;
  ba_rowstat none = {nullptr, 0, 0};
  return ba::fwd_chunk_run(q, k, v, none, o_acc, lse, o_out, B, Sq, Sk, H, H_kv, D, scale, mask_mode, causal_offset,
                           lower_offset, slopes, slopes_stride_b, dist0, pstride, nullptr, 0, 0, 0, flags, dtype,
                           stream);
}

extern "C" int ba_fwd_chunk_doc(ba_tensor4 q, ba_tensor4 k, ba_tensor4 v, ba_tensor4 o_acc, ba_rowstat lse,
                                ba_tensor4 o_out, int B, int Sq, int Sk, int H, int H_kv, int D, float scale,
                                int mask_mode, int causal_offset, int lower_offset, const int* cu_seqlens, int n_docs,
                                int64_t q_pos0, int64_t k_pos0, int pstride, int flags, int dtype, void* stream) {
  int rc;
  if ((rc = ba::check_doc_args("ba_fwd_chunk_doc", B, Sq, Sk, H, H_kv, D, scale, &mask_mode, &causal_offset,
                               &lower_offset, cu_seqlens, n_docs, q_pos0, k_pos0, pstride, dtype)))
    return rc;
  ba_rowstat none = {nullptr, 0, 0};
  return ba::fwd_chunk_run(q, k, v, none, o_acc, lse, o_out, B, Sq, Sk, H, H_kv, D, scale, mask_mode, causal_offset,
                           lower_offset, nullptr, 0, 0, pstride, cu_seqlens, n_docs, q_pos0, k_pos0, flags, dtype,
                           stream);
}
