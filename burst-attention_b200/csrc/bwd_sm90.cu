// ba_bwd_chunk*: the backward entry points, their deterministic-mode workspace, and the tile kernel without a band's
// lower edge (bwd_sm90.cuh).
#include <mutex>
#include <vector>

#include "bwd_sm90.cuh"

namespace ba {

// Deterministic-mode workspace (turn counters + tickets), one per (device, stream), grown on demand, zeroed on
// the launching stream before every launch.  Launches on one stream are ordered, so they can share a
// workspace; different streams / devices / host threads never do (a mutex guards the table).
struct BwdWorkspace {
  int device;
  cudaStream_t stream;
  int* ptr;
  size_t cap;
};
static std::mutex g_ws_mutex;
static std::vector<BwdWorkspace> g_ws;

static int* bwd_sem_workspace(size_t n_ints, cudaStream_t stream) {
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return nullptr;
  std::lock_guard<std::mutex> lock(g_ws_mutex);
  BwdWorkspace* w = nullptr;
  for (auto& e : g_ws)
    if (e.device == dev && e.stream == stream) w = &e;
  if (!w) {
    g_ws.push_back(BwdWorkspace{dev, stream, nullptr, 0});
    w = &g_ws.back();
  }
  if (w->cap < n_ints) {
    // the old buffer may still be in use by a launch in flight on this stream: free it in stream order
    if (w->ptr && cudaFreeAsync(w->ptr, stream) != cudaSuccess) return nullptr;
    w->ptr = nullptr, w->cap = 0;
    if (cudaMallocAsync(reinterpret_cast<void**>(&w->ptr), n_ints * sizeof(int), stream) != cudaSuccess) return nullptr;
    w->cap = n_ints;
  }
  if (cudaMemsetAsync(w->ptr, 0, n_ints * sizeof(int), stream) != cudaSuccess) return nullptr;
  return w->ptr;
}

// Every backward entry point after its argument check: fill BwdParams and launch the tile kernel of the call's masks.
static int bwd_chunk_run(ba_tensor4 d_o, ba_tensor4 q, ba_tensor4 k, ba_tensor4 v, ba_rowstat delta, ba_rowstat lse,
                         ba_tensor4 dq_acc, ba_tensor4 dk_acc, ba_tensor4 dv_acc, const ChunkArgs& a, int flags,
                         void* stream) {
  int rc;
  BA_REQUIRE(d_o.ptr && q.ptr && k.ptr && v.ptr && delta.ptr && lse.ptr, "ba_bwd_chunk: null input");
  BA_REQUIRE(dq_acc.ptr && dk_acc.ptr && dv_acc.ptr && aligned16(dq_acc, 4) && aligned16(dk_acc, 4) &&
                 aligned16(dv_acc, 4),
             "ba_bwd_chunk: fp32 accumulators must be non-null, 16-byte aligned, strides multiple of 4");

  CUtensorMap tmQ, tmK, tmV, tmDO, tmDQ;
  const CUtensorMapDataType dt = lowp_dtype(a.dtype);
  if ((rc = make_tensor_map(&tmQ, q, a.B, a.Sq, a.H, a.D, dt, 2, 64, kBwdM, true))) return rc;
  if ((rc = make_tensor_map(&tmDO, d_o, a.B, a.Sq, a.H, a.D, dt, 2, 64, kBwdM, true))) return rc;
  if ((rc = make_tensor_map(&tmK, k, a.B, a.Sk, a.H_kv, a.D, dt, 2, 64, kBwdN, true))) return rc;
  if ((rc = make_tensor_map(&tmV, v, a.B, a.Sk, a.H_kv, a.D, dt, 2, 64, kBwdN, true))) return rc;
  // dQ reductions: [64 rows][32 fp32 columns] SW128 boxes (two per reducing warpgroup), H query heads
  if ((rc = make_tensor_map(&tmDQ, dq_acc, a.B, a.Sq, a.H, a.D, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, 32, kBwdM, true)))
    return rc;

  BwdParams p;
  p.lse = lse.ptr, p.lse_sb = lse.stride_b, p.lse_sh = lse.stride_h;
  p.delta = delta.ptr, p.dl_sb = delta.stride_b, p.dl_sh = delta.stride_h;
  p.dk_acc = static_cast<float*>(dk_acc.ptr);
  p.dk_sb = dk_acc.stride_b, p.dk_ss = dk_acc.stride_s, p.dk_sh = dk_acc.stride_h;
  p.dv_acc = static_cast<float*>(dv_acc.ptr);
  p.dv_sb = dv_acc.stride_b, p.dv_ss = dv_acc.stride_s, p.dv_sh = dv_acc.stride_h;
  p.bias = a.key_bias.ptr, p.bias_sb = a.key_bias.stride_b, p.bias_sh = a.key_bias.stride_h;
  p.B = a.B, p.Sq = a.Sq, p.Sk = a.Sk, p.H = a.H;
  p.G = a.H / a.H_kv;
  p.scale = a.scale;
  p.scale_log2 = a.scale * kLog2e;
  p.causal = (a.mask_mode & BA_MASK_CAUSAL) != 0;
  p.causal_off = a.causal_offset;
  p.lo = a.lower_offset;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  p.sem = p.ticket = nullptr;
  if (flags & BA_BWD_DETERMINISTIC) {
    const size_t n_turn = (size_t)a.B * a.H * ((a.Sq + kBwdM - 1) / kBwdM);  // per (batch, query head, Q block)
    const size_t n = n_turn + (size_t)a.B * a.H_kv;                           // tickets per (batch, K/V head)
    p.sem = bwd_sem_workspace(n, st);
    if (p.sem) p.ticket = p.sem + n_turn;
    if (!p.sem) {
      set_error("ba_bwd_chunk: could not allocate the deterministic-mode workspace (%zu ints)", n);
      return BA_ERR_CUDA;
    }
  }
  p.slopes = a.slopes, p.slopes_sb = a.slopes_stride_b, p.dist0 = a.dist0, p.pstride = a.pstride;
  p.cu = a.cu_seqlens, p.n_docs = a.n_docs, p.q_pos0 = (int)a.q_pos0, p.k_pos0 = (int)a.k_pos0;  // checked: they fit

  const bool bf16 = a.dtype == BA_DTYPE_BF16, lower = a.mask_mode & BA_MASK_LOWER;
  const BwdKernel kern = a.cu_seqlens ? bwd_doc_kernel_of(bf16, a.D)
                         : a.slopes   ? bwd_alibi_kernel_of(bf16, a.D, lower)
                         : lower      ? bwd_band_kernel_of(bf16, a.D)
                                      : bwd_chunk_kernel_of<false>(bf16, a.D);
  BA_CHECK_CUDA(cudaFuncSetAttribute(kern.fn, cudaFuncAttributeMaxDynamicSharedMemorySize, kern.smem));
  dim3 grid((a.Sk + kBwdN - 1) / kBwdN, a.H_kv, a.B);  // one CTA per (key block, K/V head, batch)
  kern.fn<<<grid, kBwdThreads, kern.smem, st>>>(tmQ, tmK, tmV, tmDO, tmDQ, p);
  BA_CHECK_CUDA(cudaGetLastError());
  return BA_OK;
}

}  // namespace ba

extern "C" int ba_bwd_chunk(ba_tensor4 d_o, ba_tensor4 q, ba_tensor4 k, ba_tensor4 v, ba_rowstat delta,
                            ba_rowstat lse, ba_tensor4 dq_acc, ba_tensor4 dk_acc, ba_tensor4 dv_acc, int B, int Sq,
                            int Sk, int H, int D, float scale, int mask_mode, int causal_offset, int flags, int dtype,
                            void* stream) {
  ba_rowstat none = {nullptr, 0, 0};
  return ba_bwd_chunk_bias(d_o, q, k, v, delta, lse, none, dq_acc, dk_acc, dv_acc, B, Sq, Sk, H, D, scale, mask_mode,
                           causal_offset, flags, dtype, stream);
}

extern "C" int ba_bwd_chunk_bias(ba_tensor4 d_o, ba_tensor4 q, ba_tensor4 k, ba_tensor4 v, ba_rowstat delta,
                                 ba_rowstat lse, ba_rowstat key_bias, ba_tensor4 dq_acc, ba_tensor4 dk_acc,
                                 ba_tensor4 dv_acc, int B, int Sq, int Sk, int H, int D, float scale, int mask_mode,
                                 int causal_offset, int flags, int dtype, void* stream) {
  return ba_bwd_chunk_gqa(d_o, q, k, v, delta, lse, key_bias, dq_acc, dk_acc, dv_acc, B, Sq, Sk, H, H, D, scale,
                          mask_mode, causal_offset, flags, dtype, stream);
}

extern "C" int ba_bwd_chunk_gqa(ba_tensor4 d_o, ba_tensor4 q, ba_tensor4 k, ba_tensor4 v, ba_rowstat delta,
                                ba_rowstat lse, ba_rowstat key_bias, ba_tensor4 dq_acc, ba_tensor4 dk_acc,
                                ba_tensor4 dv_acc, int B, int Sq, int Sk, int H, int H_kv, int D, float scale,
                                int mask_mode, int causal_offset, int flags, int dtype, void* stream) {
  ba::ChunkArgs a{B, Sq, Sk, H, H_kv, D, scale, mask_mode, causal_offset, 0, dtype};
  a.key_bias = key_bias;
  const int rc = ba::check_chunk_args("ba_bwd_chunk", ba::ChunkEntry::kPlain, &a);
  return rc ? rc : ba::bwd_chunk_run(d_o, q, k, v, delta, lse, dq_acc, dk_acc, dv_acc, a, flags, stream);
}

extern "C" int ba_bwd_chunk_band(ba_tensor4 d_o, ba_tensor4 q, ba_tensor4 k, ba_tensor4 v, ba_rowstat delta,
                                 ba_rowstat lse, ba_rowstat key_bias, ba_tensor4 dq_acc, ba_tensor4 dk_acc,
                                 ba_tensor4 dv_acc, int B, int Sq, int Sk, int H, int H_kv, int D, float scale,
                                 int mask_mode, int causal_offset, int lower_offset, int flags, int dtype,
                                 void* stream) {
  ba::ChunkArgs a{B, Sq, Sk, H, H_kv, D, scale, mask_mode, causal_offset, lower_offset, dtype};
  a.key_bias = key_bias;
  const int rc = ba::check_chunk_args("ba_bwd_chunk", ba::ChunkEntry::kBand, &a);
  return rc ? rc : ba::bwd_chunk_run(d_o, q, k, v, delta, lse, dq_acc, dk_acc, dv_acc, a, flags, stream);
}

extern "C" int ba_bwd_chunk_alibi(ba_tensor4 d_o, ba_tensor4 q, ba_tensor4 k, ba_tensor4 v, ba_rowstat delta,
                                  ba_rowstat lse, ba_tensor4 dq_acc, ba_tensor4 dk_acc, ba_tensor4 dv_acc, int B, int Sq,
                                  int Sk, int H, int H_kv, int D, float scale, int mask_mode, int causal_offset,
                                  int lower_offset, const float* slopes, int64_t slopes_stride_b, int64_t dist0,
                                  int pstride, int flags, int dtype, void* stream) {
  ba::ChunkArgs a{B, Sq, Sk, H, H_kv, D, scale, mask_mode, causal_offset, lower_offset, dtype};
  a.slopes = slopes, a.slopes_stride_b = slopes_stride_b, a.dist0 = dist0, a.pstride = pstride;
  const int rc = ba::check_chunk_args("ba_bwd_chunk_alibi", ba::ChunkEntry::kAlibi, &a);
  return rc ? rc : ba::bwd_chunk_run(d_o, q, k, v, delta, lse, dq_acc, dk_acc, dv_acc, a, flags, stream);
}

extern "C" int ba_bwd_chunk_doc(ba_tensor4 d_o, ba_tensor4 q, ba_tensor4 k, ba_tensor4 v, ba_rowstat delta,
                                ba_rowstat lse, ba_tensor4 dq_acc, ba_tensor4 dk_acc, ba_tensor4 dv_acc, int B, int Sq,
                                int Sk, int H, int H_kv, int D, float scale, int mask_mode, int causal_offset,
                                int lower_offset, const int* cu_seqlens, int n_docs, int64_t q_pos0, int64_t k_pos0,
                                int pstride, int flags, int dtype, void* stream) {
  ba::ChunkArgs a{B, Sq, Sk, H, H_kv, D, scale, mask_mode, causal_offset, lower_offset, dtype};
  a.cu_seqlens = cu_seqlens, a.n_docs = n_docs, a.q_pos0 = q_pos0, a.k_pos0 = k_pos0, a.pstride = pstride;
  const int rc = ba::check_chunk_args("ba_bwd_chunk_doc", ba::ChunkEntry::kDoc, &a);
  return rc ? rc : ba::bwd_chunk_run(d_o, q, k, v, delta, lse, dq_acc, dk_acc, dv_acc, a, flags, stream);
}
