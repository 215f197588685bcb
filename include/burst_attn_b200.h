/* burst_attn_b200 -- C ABI of the H100-native (sm_90a) chunk operators and ring transport
 * that replace the reference's "operator boundary" (SURVEY.md 8b):
 *
 *   attn_forward / attn_backward      burst_attn/burst_attn_interface.py:40-93
 *   inter_flash_cuda_fwd / _bwd       burst_attn/burst_utils.py:149-249
 *   cuda_scale_out_lse_helper (merge) burst_attn/burst_utils.py:20-33   (fused into ba_fwd_chunk)
 *   delta = rowsum(O*dO)              burst_attn/burst_attn_interface.py:272-278
 *   Ring.{double_ring_send_recv,commit,wait}   burst_attn/comm.py:221-321
 *
 * Plain C: pointers, sizes, strides (in ELEMENTS), a cudaStream_t passed as void*.
 * Every function returns 0 on success, non-zero on error; ba_last_error() gives
 * a human-readable message for the calling thread.  Nothing here allocates
 * device memory on the hot path and nothing synchronises the host.
 *
 * Layout: tensors are addressed as [b, s, h, d] through explicit strides with
 * d contiguous, so both the reference's flash layout [B,S,H,D] and its
 * "normal" layout [B,H,S,D] are expressible, as are half-sequence / shifted
 * views (base pointer + length) without copies.
 */
#ifndef BURST_ATTN_B200_H
#define BURST_ATTN_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define BA_OK 0
#define BA_ERR_INVALID 1
#define BA_ERR_CUDA 2
#define BA_ERR_NCCL 3
#define BA_ERR_UNSUPPORTED 4

/* element types of q/k/v/dO and of the low-precision output */
#define BA_DTYPE_FP16 0
#define BA_DTYPE_BF16 1

/* mask modes (SURVEY.md Appendix B) */
#define BA_MASK_NONE 0
#define BA_MASK_CAUSAL 1 /* key j visible to query i iff j <= i + causal_offset */
#define BA_MASK_LOWER 2  /* band entry points only: key j visible to query i only if j >= i + lower_offset */

/* flags for ba_fwd_chunk */
#define BA_FWD_FIRST 1 /* no carried state: start from (O=0, lse=-inf)                       */
#define BA_FWD_LAST 2  /* write the normalised output in the input dtype to o_out             */

/* flags for ba_bwd_chunk */
#define BA_BWD_DETERMINISTIC 1 /* dQ reduced in key-block order (bitwise reproducible, slower)   */

/* A [b,s,h,d] view: d is contiguous, the other strides are in elements. */
typedef struct {
  void* ptr;
  int64_t stride_b;
  int64_t stride_s;
  int64_t stride_h;
} ba_tensor4;

/* A [b,h,s] fp32 view (lse, delta): s is contiguous. */
typedef struct {
  float* ptr;
  int64_t stride_b;
  int64_t stride_h;
} ba_rowstat;

const char* ba_last_error(void);
/* Library / device capability probe: returns BA_OK when the current device is sm_90 (H100). */
int ba_device_check(void);
int ba_version(void);

/* One ring round of the forward (replaces attn_forward(flash="cuda"),
 * burst_attn_interface.py:40-51 -> inter_flash_cuda_fwd, burst_utils.py:149-177,
 * including the separate LSE-merge launches of cuda_scale_out_lse_helper):
 * attends q[B,Sq,H,D] to one K/V chunk [B,Sk,H,D] and folds the result into the
 * running state (o_acc fp32, already normalised; lse fp32 [B,H,Sq]).
 *   flags & BA_FWD_FIRST : state is not read.
 *   flags & BA_FWD_LAST  : o_out (dtype) is written instead of o_acc; lse is always written.
 * D must be 64 or 128; Sq, Sk arbitrary (>0).  scale > 0.                        */
int ba_fwd_chunk(ba_tensor4 q, ba_tensor4 k, ba_tensor4 v, ba_tensor4 o_acc, ba_rowstat lse, ba_tensor4 o_out,
                 int B, int Sq, int Sk, int H, int D, float scale, int mask_mode, int causal_offset, int flags,
                 int dtype, void* stream);

/* The same with an additive attention bias per KEY: scores = q k^T * scale + key_bias[b,h,key]  (the "vector" bias
 * of the reference's LAO tile, burst_attn/lao.py:102-105,155-173; its ring op always passes bias = None,
 * burst_attn_interface.py:223,316, so this serves the single-GPU wrappers of burst_attn/flash_triton.py).
 * key_bias: fp32 [B,H,Sk] view (stride_b may be 0 to broadcast over the batch; ptr NULL = no bias).  -inf entries
 * mask a key.  Both kernels add it in the exponent's FMA; no gradient is produced for the bias (neither does the
 * reference: flash_triton.py:1046).                                                                              */
int ba_fwd_chunk_bias(ba_tensor4 q, ba_tensor4 k, ba_tensor4 v, ba_rowstat key_bias, ba_tensor4 o_acc, ba_rowstat lse,
                      ba_tensor4 o_out, int B, int Sq, int Sk, int H, int D, float scale, int mask_mode,
                      int causal_offset, int flags, int dtype, void* stream);

/* Grouped-query attention (GQA; MQA when H_kv == 1): the same as ba_fwd_chunk_bias with k, v of H_kv heads
 * ([B,Sk,H_kv,D]).  Query head h attends with K/V head h / (H / H_kv); H % H_kv == 0 and H_kv > 0 are required.
 * H applies to q, o_acc, o_out, lse and key_bias; H_kv to k and v.  H_kv == H is ba_fwd_chunk_bias.        */
int ba_fwd_chunk_gqa(ba_tensor4 q, ba_tensor4 k, ba_tensor4 v, ba_rowstat key_bias, ba_tensor4 o_acc, ba_rowstat lse,
                     ba_tensor4 o_out, int B, int Sq, int Sk, int H, int H_kv, int D, float scale, int mask_mode,
                     int causal_offset, int flags, int dtype, void* stream);

/* Band mask (sliding-window / local attention): the same as ba_fwd_chunk_gqa with mask_mode a set of bits,
 * BA_MASK_CAUSAL (key j visible to query i only if j <= i + causal_offset) and BA_MASK_LOWER (only if
 * j >= i + lower_offset); either side may be open.  With both bits lower_offset <= causal_offset is required.  A row
 * that sees no key has lse = -inf and O = 0 (or keeps its carried state).  The CTA of a 128-row Q tile loads only the
 * K/V tiles its band reaches.  ba_fwd_chunk_gqa is this call with BA_MASK_LOWER clear.                        */
int ba_fwd_chunk_band(ba_tensor4 q, ba_tensor4 k, ba_tensor4 v, ba_rowstat key_bias, ba_tensor4 o_acc, ba_rowstat lse,
                      ba_tensor4 o_out, int B, int Sq, int Sk, int H, int H_kv, int D, float scale, int mask_mode,
                      int causal_offset, int lower_offset, int flags, int dtype, void* stream);

/* ALiBi (linear position bias): ba_fwd_chunk_band without a key bias, plus the bias -slope |d| added to the scores of
 * row i and key j (before the softmax), with the distance d = pstride (i - j) + dist0 counted in exact integers.
 * slopes: fp32, one per query head, of batch b at slopes + b * slopes_stride_b (0: one row for every batch).  A ring
 * passes dist0 = the full-sequence position of row 0 minus that of key 0, and pstride = the distance in the full
 * sequence between neighbouring rows (1, or W for a striped shard).  pstride >= 1.                               */
int ba_fwd_chunk_alibi(ba_tensor4 q, ba_tensor4 k, ba_tensor4 v, ba_tensor4 o_acc, ba_rowstat lse, ba_tensor4 o_out,
                       int B, int Sq, int Sk, int H, int H_kv, int D, float scale, int mask_mode, int causal_offset,
                       int lower_offset, const float* slopes, int64_t slopes_stride_b, int64_t dist0, int pstride,
                       int flags, int dtype, void* stream);

/* Packed documents (flash-attn's cu_seqlens): ba_fwd_chunk_band without a key bias, where row i and key j also see
 * each other only inside one document.  cu_seqlens: device int32, n_docs + 1 non-decreasing boundaries of the full
 * sequence from cu_seqlens[0] = 0 (repeated values are zero-length documents); document d holds the positions
 * [cu_seqlens[d], cu_seqlens[d + 1]).  Row i sits at position q_pos0 + pstride i and key j at k_pos0 + pstride j (a
 * ring passes each launch's own; pstride is W for a striped shard, else 1).  A row with no visible key keeps its
 * carried state (lse = -inf and O = 0 without one).  n_docs >= 1, pstride >= 1, q_pos0, k_pos0 >= 0.            */
int ba_fwd_chunk_doc(ba_tensor4 q, ba_tensor4 k, ba_tensor4 v, ba_tensor4 o_acc, ba_rowstat lse, ba_tensor4 o_out,
                     int B, int Sq, int Sk, int H, int H_kv, int D, float scale, int mask_mode, int causal_offset,
                     int lower_offset, const int* cu_seqlens, int n_docs, int64_t q_pos0, int64_t k_pos0, int pstride,
                     int flags, int dtype, void* stream);

/* delta[b,h,s] = sum_d O[b,s,h,d] * dO[b,s,h,d]  (burst_attn_interface.py:272-278) */
int ba_bwd_delta(ba_tensor4 o, ba_tensor4 d_o, ba_rowstat delta, int B, int S, int H, int D, int dtype,
                 void* stream);

/* One ring round of the backward (replaces attn_backward(flash="cuda"),
 * burst_attn_interface.py:54-93 -> inter_flash_cuda_bwd, burst_utils.py:180-249,
 * plus the three "+=" passes of burst_attn_interface.py:379-390): for the
 * Q-bundle (q, dO, delta, lse) against the home K/V chunk, ACCUMULATES
 *   dq_acc[B,Sq,H,D] += dS K,  dk_acc[B,Sk,H,D] += dS^T Q,  dv_acc[B,Sk,H,D] += P^T dO
 * into fp32 accumulators.                                                          */
int ba_bwd_chunk(ba_tensor4 d_o, ba_tensor4 q, ba_tensor4 k, ba_tensor4 v, ba_rowstat delta, ba_rowstat lse,
                 ba_tensor4 dq_acc, ba_tensor4 dk_acc, ba_tensor4 dv_acc, int B, int Sq, int Sk, int H, int D,
                 float scale, int mask_mode, int causal_offset, int flags, int dtype, void* stream);

int ba_bwd_chunk_bias(ba_tensor4 d_o, ba_tensor4 q, ba_tensor4 k, ba_tensor4 v, ba_rowstat delta, ba_rowstat lse,
                      ba_rowstat key_bias, ba_tensor4 dq_acc, ba_tensor4 dk_acc, ba_tensor4 dv_acc, int B, int Sq, int Sk,
                      int H, int D, float scale, int mask_mode, int causal_offset, int flags, int dtype, void* stream);

/* Grouped-query attention: the same as ba_bwd_chunk_bias with k, v, dk_acc, dv_acc of H_kv heads.  dK / dV of a
 * K/V head accumulate the sum over its H / H_kv query heads.  H applies to q, d_o, delta, lse, key_bias and dq_acc.
 * H % H_kv == 0 and H_kv > 0 are required; H_kv == H is ba_bwd_chunk_bias.                                      */
int ba_bwd_chunk_gqa(ba_tensor4 d_o, ba_tensor4 q, ba_tensor4 k, ba_tensor4 v, ba_rowstat delta, ba_rowstat lse,
                     ba_rowstat key_bias, ba_tensor4 dq_acc, ba_tensor4 dk_acc, ba_tensor4 dv_acc, int B, int Sq, int Sk,
                     int H, int H_kv, int D, float scale, int mask_mode, int causal_offset, int flags, int dtype,
                     void* stream);

/* Band mask: the same as ba_bwd_chunk_gqa with the mask bits and lower_offset of ba_fwd_chunk_band.  The CTA of a
 * 128-key block visits only the 64-row Q blocks whose band reaches it; keys no row sees get dK = dV = 0 added.
 * BA_BWD_DETERMINISTIC stays bitwise reproducible.  ba_bwd_chunk_gqa is this call with BA_MASK_LOWER clear.      */
int ba_bwd_chunk_band(ba_tensor4 d_o, ba_tensor4 q, ba_tensor4 k, ba_tensor4 v, ba_rowstat delta, ba_rowstat lse,
                      ba_rowstat key_bias, ba_tensor4 dq_acc, ba_tensor4 dk_acc, ba_tensor4 dv_acc, int B, int Sq,
                      int Sk, int H, int H_kv, int D, float scale, int mask_mode, int causal_offset, int lower_offset,
                      int flags, int dtype, void* stream);

/* ALiBi: ba_bwd_chunk_band without a key bias, plus the bias of ba_fwd_chunk_alibi.  No gradient flows into the
 * slopes.                                                                                                        */
int ba_bwd_chunk_alibi(ba_tensor4 d_o, ba_tensor4 q, ba_tensor4 k, ba_tensor4 v, ba_rowstat delta, ba_rowstat lse,
                       ba_tensor4 dq_acc, ba_tensor4 dk_acc, ba_tensor4 dv_acc, int B, int Sq, int Sk, int H, int H_kv,
                       int D, float scale, int mask_mode, int causal_offset, int lower_offset, const float* slopes,
                       int64_t slopes_stride_b, int64_t dist0, int pstride, int flags, int dtype, void* stream);

/* Packed documents: ba_bwd_chunk_band without a key bias, with the documents of ba_fwd_chunk_doc.  A key block
 * visits only the Q blocks of its documents; keys no row shares a document with get dK = dV = 0 added.
 * BA_BWD_DETERMINISTIC stays bitwise reproducible.                                                               */
int ba_bwd_chunk_doc(ba_tensor4 d_o, ba_tensor4 q, ba_tensor4 k, ba_tensor4 v, ba_rowstat delta, ba_rowstat lse,
                     ba_tensor4 dq_acc, ba_tensor4 dk_acc, ba_tensor4 dv_acc, int B, int Sq, int Sk, int H, int H_kv,
                     int D, float scale, int mask_mode, int causal_offset, int lower_offset, const int* cu_seqlens,
                     int n_docs, int64_t q_pos0, int64_t k_pos0, int pstride, int flags, int dtype, void* stream);

/* dst[b,s,h,d] (dtype) = src[b,s,h,d] (fp32); used once per backward to hand the
 * fp32 gradient accumulators back in the input dtype.                              */
int ba_cast_from_f32(ba_tensor4 src, ba_tensor4 dst, int B, int S, int H, int D, int dtype, void* stream);
/* dst (fp32) += src (fp32): dQ ring add-on-arrival (comm.py:202).                   */
int ba_accumulate_f32(ba_tensor4 src, ba_tensor4 dst, int B, int S, int H, int D, void* stream);

/* ---- ring transport (replaces comm.py Ring, single-ring path) -------------------
 * A ring owns one NCCL communicator and one side stream.  ba_ring_post enqueues,
 * on the side stream, a grouped ncclSend(src[i] -> next) / ncclRecv(dst[i] <- prev)
 * after an event recorded on `compute_stream` (data dependencies of the sources);
 * ba_ring_wait makes `compute_stream` wait for the posted transfers.  No host sync. */
typedef struct ba_ring ba_ring;
#define BA_NCCL_UNIQUE_ID_BYTES 128
int ba_ring_unique_id(void* out_id128);
int ba_ring_create(const void* id128, int rank, int world, ba_ring** out);
int ba_ring_post(ba_ring* ring, const void* const* src, void* const* dst, const int64_t* nbytes, int n,
                 void* compute_stream);
int ba_ring_wait(ba_ring* ring, void* compute_stream);
int ba_ring_rank(const ba_ring* ring);
int ba_ring_world(const ba_ring* ring);
int ba_ring_destroy(ba_ring* ring);

/* ---- copy-engine transport of a ring (optional; rings whose ranks share a node) ----
 * NCCL's send/recv are SM-resident kernels that compete with the tile kernels; for short shards that
 * exposes the hop.  A ring can instead own a RECEIVE ARENA: one device allocation per rank, carved
 * identically on every rank (destination i of a post has the same offset everywhere), mapped into both
 * neighbours with CUDA IPC.  Once connected, ba_ring_post pushes each source into the next rank's arena
 * with peer cudaMemcpyAsync (copy engines over NVLink, zero SMs) and flow-controls with two hop counters
 * per rank awaited by cuStreamWaitValue32 -- same post/wait contract, still no host synchronisation.
 *   ba_ring_arena_create : (re)allocates the local arena of `bytes` data bytes; returns its data base and
 *                          a 64-byte IPC handle to hand to both neighbours (any host channel).  All ranks
 *                          must be quiescent (device-synchronised + barrier) when an arena is replaced.
 *   ba_ring_arena_connect: maps the previous and the next rank's arenas (and frees a replaced arena).  Call it
 *                          only after a collective that follows every rank's ba_ring_arena_create.  From here on every destination
 *                          passed to ba_ring_post must lie inside the local arena.
 * A ring created with id128 == NULL has no NCCL communicator and must be connected before its first post. */
#define BA_IPC_HANDLE_BYTES 64
int ba_ring_arena_create(ba_ring* ring, int64_t bytes, void** base_out, void* handle_out64);
int ba_ring_arena_connect(ba_ring* ring, const void* prev_handle64, const void* next_handle64);

#ifdef __cplusplus
}
#endif
#endif /* BURST_ATTN_B200_H */
