// ba_fwd_chunk: one ring round of the forward on sm_90a.
//
// Replaces, for flash="cuda"/"triton", the reference's per-round
//   flash_attn_2_cuda.fwd  +  cuda_scale_out_lse_helper          (burst_utils.py:149-177, :20-33)
// and the Triton LAO tile with carried state                       (lao.py:66-244)
// by ONE kernel: the carried (O fp32 normalised, lse) state is loaded in the
// prologue as the initial online-softmax state (m = lse, l = 1, acc = O) and the
// merged state is written in the epilogue -- no separate merge pass over HBM.
//
// Grouped-query attention: K/V may have H / G heads; query head h reads K/V head h / G.  The grid is
// (Q tiles, query heads, batch), so the G query heads of a group are adjacent in blockIdx.y and their CTAs sweep
// the same K/V slice while it is resident in L2.
//
// Structure (one CTA = one 128-row Q tile of one (batch, head)):
//   warpgroup 0   one TMA producer thread: Q once, then K_i / V_i tiles into 2-stage rings (and, with a key bias,
//                 the tile's bias in log2 units); the other warps of the group only hand their registers over
//   warpgroups 1, 2  64 Q rows each, everything in registers:
//                 S = Q_w K_i^T      (wgmma SS m64n128, both operands K-major SW128 smem)
//                 online softmax     (a thread owns 2 rows x 32 columns of S; row reductions over the quad)
//                 O_w += P V_i       (wgmma RS: P re-packed to 16 bit in registers as the A operand, V MN-major)
// The two consumer warpgroups run unsynchronised, so one group's softmax overlaps the other's MMAs.
//
// Band mask (kBand, sliding-window attention): key c is visible to row a iff a + lo <= c, on top of the upper edge
// c <= a + causal_off when causal.  A CTA then visits the tiles [t0, t0 + n_tiles): the first is the tile of the
// first row's lowest visible key, so tiles entirely below the band of all its rows are never loaded, and each
// consumer warpgroup works on its own sub-range of them.  kBand = false is the kernel without a lower edge; its
// instantiations live in fwd_sm90.cu, the kBand = true ones in fwd_band_sm90.cu.
//
// ALiBi (kAlibi, fwd_alibi_kernel in fwd_alibi_sm90.cu): the score of row a and key c gets -slope |pstride (a - c) +
// dist0|, formed from exact integer distances relative to each row's reference (alibi_dref); tiles and masks are
// unchanged.
//
// Packed documents (kDoc, fwd_doc_kernel in fwd_doc_sm90.cu; always with kBand): row a and key c see each other only
// inside one document of cu_seqlens, on top of the band.  Within a launch positions are affine in a and c, so each
// row's keys of its document are one interval of the view, intersected with the row's band limits; each warpgroup's
// tile range is narrowed to the document intervals of its first and last row, and the CTA visits the hull of the two.
#pragma once
#include <math.h>
#include <stdlib.h>

#include "doc_sm90.cuh"
#include "host_common.h"
#include "sm90_ptx.cuh"

namespace ba {

constexpr int kBlockM = 128;  // Q rows per CTA (64 per consumer warpgroup)
constexpr int kBlockN = 128;  // keys per K/V tile
constexpr int kKStages = 2;
constexpr int kVStages = 2;
constexpr int kBoxBytes = 128 * 64 * 2;  // 16 KiB: one 128 x 64 SW128 TMA box (a [128][head_dim] tile is head_dim/64 boxes)
constexpr int kFwdThreads = 384;         // warpgroup 0: TMA producer; warpgroups 1, 2: MMA + softmax

struct FwdParams {
  float* o_acc;
  int64_t oacc_sb, oacc_ss, oacc_sh;
  float* lse;
  int64_t lse_sb, lse_sh;
  void* o_out;
  int64_t oout_sb, oout_ss, oout_sh;
  int B, Sq, Sk, H;
  int G;              // query heads per K/V head (grouped-query attention; 1 = MHA): head h reads K/V head h / G
  float scale_log2;
  const float* bias;  // optional additive bias per key [B|1, H, Sk] (fp32, indexed by the query head), or null
  int64_t bias_sb, bias_sh;
  int causal;
  int causal_off;
  int load_state;
  int store_lowp;
  int lo;  // kBand: key c is visible to row a only if c >= a + lo
  // kAlibi (appended, so the fields above keep their offsets): row a and key c get the bias -slope |d| with the
  // exact integer distance d = pstride (a - c) + dist0; slope = slopes[b * slopes_sb + h] (query head)
  const float* slopes;
  int64_t slopes_sb;
  int64_t dist0;
  int pstride;  // ALiBi and kDoc: the distance in the full sequence between neighbouring rows (and keys)
  // kDoc (appended): row a sits at position q_pos0 + pstride a, key c at k_pos0 + pstride c; both see each other only
  // inside one document [cu[d], cu[d + 1]) of the n_docs + 1 boundaries cu (device int32; every position fits)
  const int* cu;
  int n_docs;
  int q_pos0, k_pos0;
};

struct __align__(8) FwdBarriers {
  uint64_t q_full;
  uint64_t k_full[kKStages], k_empty[kKStages];
  uint64_t b_full[kKStages];  // kBias: the key-bias row of this K stage has been written
  uint64_t v_full[kVStages], v_empty[kVStages];
};

// shared-memory carve-up for head dim kD (64 or 128): a tile is [128 rows][kD] 16-bit = kD/64 SW128 boxes of
// [128 rows][64 cols] (16 KiB each)
template <int kD>
struct FwdLayout {
  static_assert(kD == 64 || kD == 128, "head dim 64 or 128");
  static constexpr uint32_t kTileB = 128 * kD * 2;
  static constexpr int kBoxes = kD / 64;
  static constexpr uint32_t kOffQ = 0;
  static constexpr uint32_t kOffK = kTileB;
  static constexpr uint32_t kOffV = kOffK + kKStages * kTileB;
  static constexpr uint32_t kOffBias = kOffV + kVStages * kTileB;  // [kKStages][128] fp32
  static constexpr uint32_t kOffBars = kOffBias + kKStages * kBlockN * 4;
  static constexpr int kSmemBytes = kOffBars + 256 /*barriers*/;
  static_assert(kSmemBytes <= 232448, "forward kernel exceeds 227 KiB of shared memory");
};

// number of 128-key tiles the 64 Q rows starting at r0 must visit
__device__ __forceinline__ int fwd_trip_count(int r0, const FwdParams& p) {
  if (r0 >= p.Sq) return 0;
  int r_last = min(r0 + 63, p.Sq - 1);
  int max_limit = p.causal ? min(r_last + p.causal_off, p.Sk - 1) : p.Sk - 1;
  return max_limit < 0 ? 0 : max_limit / kBlockN + 1;
}

// band: the first 128-key tile the 64 Q rows starting at r0 must visit (the tile of row r0's lowest visible key;
// the host clamps lo to <= Sk, so r0 + lo does not overflow)
__device__ __forceinline__ int fwd_first_tile(int r0, const FwdParams& p) { return max(0, r0 + p.lo) / kBlockN; }

// kDoc: the 128-key tiles [*first, *end) the 64 Q rows starting at r0 must visit: the band's tiles narrowed to the
// keys that share a document with the first row (from below) and the last row (from above); [0, 0) when none.
// Documents never decrease along the rows, so these two bound the keys of every row in between.
__device__ __forceinline__ void fwd_doc_range(int r0, const FwdParams& p, int* first, int* end) {
  *first = *end = 0;
  if (r0 >= p.Sq) return;
  const int r_last = min(r0 + 63, p.Sq - 1);
  int k_lo, k_hi, unused;
  doc_interval(p.q_pos0 + p.pstride * r0, p.cu, p.n_docs, p.k_pos0, p.pstride, p.Sk, &k_lo, &unused);
  doc_interval(p.q_pos0 + p.pstride * r_last, p.cu, p.n_docs, p.k_pos0, p.pstride, p.Sk, &unused, &k_hi);
  const int f = max(fwd_first_tile(r0, p), k_lo / kBlockN);
  const int e = min(fwd_trip_count(r0, p), (k_hi + kBlockN - 1) / kBlockN);
  if (e > f) *first = f, *end = e;
}

// ALiBi: the smallest |d| of row a over the view's keys 0 .. Sk-1 (0 if d changes sign).  The kernel runs the row's
// softmax relative to the bias -slope dref, so that far from d = 0 its fp32 scores stay small: a pair's score gets
// -slope (|d| - dref), an exact integer times the slope, and only lse carries -slope dref.  A carried state lowers
// dref (alibi_carried_ref) so that its lse, taken to the row's reference, stays small too.
__device__ __forceinline__ int64_t alibi_dref(int a, const FwdParams& p) {
  const int64_t hi = (int64_t)p.pstride * a + p.dist0, lo = hi - (int64_t)p.pstride * (p.Sk - 1);
  return max((int64_t)0, max(lo, -hi));
}

// ALiBi with a carried state of lse m0 (log2 units): the reference is lowered to at most max(0, -m0) / slope, so that
// the carried state in the row's frame, m0 + slope dref, is at most max(m0, 0) and its fp32 rounding is that of m0
// itself rather than of slope dref.  Any dref <= the smallest |d| is exact (every |d| - dref stays a non-negative
// integer); keys it leaves far below the carried state only underflow to 0, as they would anyway.
__device__ __forceinline__ int64_t alibi_carried_ref(int64_t dref, float m0, float slope2) {
  if (slope2 > 0.f) {
    const float cap = fmaxf(0.f, -m0) / slope2;
    if (cap < (float)dref) return (int64_t)cap;
  }
  return dref;
}

// The kernel body; fwd_chunk_kernel (kAlibi = false), fwd_alibi_kernel (kAlibi = true, no key bias) and
// fwd_doc_kernel (kDoc = true with kBand, no key bias) wrap it.
template <bool kBF16, int kD, bool kBias, bool kBand, bool kAlibi, bool kDoc = false>
__device__ __forceinline__ void fwd_chunk_body(const CUtensorMap& tmQ, const CUtensorMap& tmK, const CUtensorMap& tmV,
                                               const FwdParams& p) {
  static_assert(!(kBias && kAlibi), "ALiBi is not combined with the key bias");
  static_assert(!kDoc || (kBand && !kBias && !kAlibi), "documents run on the band path, without key bias or ALiBi");
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = smem_raw;
  if ((smem_u32(smem) & 1023u) != 0) __trap();      // SWIZZLE_128B atoms need a 1 KiB-aligned base
  using L = FwdLayout<kD>;
  constexpr uint32_t kTileBytes = L::kTileB;
  constexpr int kBoxes = L::kBoxes, kOReg = kD / 2;  // fp32 accumulator registers of O per thread
  uint8_t* sQ = smem + L::kOffQ;
  uint8_t* sK = smem + L::kOffK;                    // [kKStages][tile]
  uint8_t* sV = smem + L::kOffV;                    // [kVStages][tile]
  float* sBias = reinterpret_cast<float*>(smem + L::kOffBias);
  FwdBarriers* bars = reinterpret_cast<FwdBarriers*>(smem + L::kOffBars);

  const int warp = __shfl_sync(0xffffffffu, threadIdx.x >> 5, 0);
  const int lane = threadIdx.x & 31;
  const int h = blockIdx.y, b = blockIdx.z;
  // causal: the last Q tiles see the most keys -- schedule them first (longest-processing-time order)
  const int row0 = (p.causal ? (int)(gridDim.x - 1 - blockIdx.x) : (int)blockIdx.x) * kBlockM;
  int n_tiles = max(fwd_trip_count(row0, p), fwd_trip_count(row0 + 64, p));
  // band: the CTA's tiles are [t0, t0 + n_tiles).  Its first warpgroup's band starts no later than the second's, and
  // with lo <= causal_off the two ranges touch, so their union is one range.
  int t0 = 0;
  if constexpr (kBand) {
    t0 = min(fwd_first_tile(row0, p), n_tiles);
    n_tiles -= t0;
  }
  // documents: the hull of the two warpgroups' ranges; a tile in a gap between them is skipped by both (`work`)
  if constexpr (kDoc) {
    int f0, e0, f1, e1;
    fwd_doc_range(row0, p, &f0, &e0);
    fwd_doc_range(row0 + 64, p, &f1, &e1);
    t0 = e0 > f0 ? (e1 > f1 ? min(f0, f1) : f0) : f1;
    n_tiles = max(0, max(e0, e1) - t0);
  }

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmQ);
    tma_prefetch_desc(&tmK);
    tma_prefetch_desc(&tmV);
    mbar_init(&bars->q_full, 1);
    for (int i = 0; i < kKStages; ++i) {
      mbar_init(&bars->k_full[i], 1);
      mbar_init(&bars->k_empty[i], 8);  // one elected arrive per consumer warp
      mbar_init(&bars->b_full[i], 1);
    }
    for (int i = 0; i < kVStages; ++i) {
      mbar_init(&bars->v_full[i], 1);
      mbar_init(&bars->v_empty[i], 8);
    }
    fence_mbar_init();
  }
  __syncthreads();

  if (warp < 4) {
    // ============================================================ TMA producer (warp 0)
    reg_alloc_dec<40>();
    if (warp != 0) return;
    const int hk = h / p.G;  // K/V head of this query head
    if (lane == 0) {
      mbar_arrive_expect_tx(&bars->q_full, kTileBytes);
      for (int half = 0; half < kBoxes; ++half)
        tma_load_4d(sQ + half * kBoxBytes, &tmQ, &bars->q_full, half * 64, h, row0, b);
    }
    for (int i = 0; i < n_tiles; ++i) {  // pipeline step i loads key tile t0 + i
      const int ks = i % kKStages, kph = (i / kKStages) & 1;
      mbar_wait(&bars->k_empty[ks], kph ^ 1);
      if (lane == 0) {
        mbar_arrive_expect_tx(&bars->k_full[ks], kTileBytes);
        for (int half = 0; half < kBoxes; ++half)
          tma_load_4d(sK + ks * kTileBytes + half * kBoxBytes, &tmK, &bars->k_full[ks], half * 64, hk,
                      (t0 + i) * kBlockN, b);
      }
      if constexpr (kBias) {  // the stage's key bias in log2 units: lane handles keys lane + 32 j
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const int key = (t0 + i) * kBlockN + lane + 32 * j;
          float x = 0.f;
          if (key < p.Sk) x = __ldg(p.bias + (int64_t)b * p.bias_sb + (int64_t)h * p.bias_sh + key) * kLog2e;
          sBias[ks * kBlockN + lane + 32 * j] = x;
        }
        __syncwarp();
        if (lane == 0) mbar_arrive(&bars->b_full[ks]);
      }
      if (lane == 0) {
        const int vs = i % kVStages, vph = (i / kVStages) & 1;
        mbar_wait(&bars->v_empty[vs], vph ^ 1);
        mbar_arrive_expect_tx(&bars->v_full[vs], kTileBytes);
        for (int half = 0; half < kBoxes; ++half)
          tma_load_4d(sV + vs * kTileBytes + half * kBoxBytes, &tmV, &bars->v_full[vs], half * 64, hk,
                      (t0 + i) * kBlockN, b);
      }
      __syncwarp();
    }
    return;
  }

  // ============================================================ consumers
  reg_alloc_inc<232>();
  const int wg = (threadIdx.x >> 7) - 1;  // 64-row half of the Q tile
  const int w = warp & 3, g = lane >> 2, t = lane & 3;
  const int r_lo = row0 + wg * 64 + 16 * w + g;  // this thread's two rows: r_lo and r_lo + 8
  const int rows[2] = {r_lo, r_lo + 8};
  // documents: this group's tiles [doc_first, doc_end) (fwd_doc_range), and each row's document keys
  [[maybe_unused]] int doc_first = 0, doc_end = 0, doc_lo[2] = {0, 0}, doc_hi[2] = {0, 0};
  if constexpr (kDoc) {
    fwd_doc_range(row0 + wg * 64, p, &doc_first, &doc_end);
#pragma unroll
    for (int r = 0; r < 2; ++r)  // a padding row (>= Sq) keeps [0, 0): its position may not fit in int32
      if (rows[r] < p.Sq)
        doc_interval(p.q_pos0 + p.pstride * rows[r], p.cu, p.n_docs, p.k_pos0, p.pstride, p.Sk, &doc_lo[r], &doc_hi[r]);
  }
  // this group's tiles end here (absolute tile index)
  const int n_mine = kDoc ? doc_end : fwd_trip_count(row0 + wg * 64, p);
  const float scale_log2 = p.scale_log2;
  int limit[2];
#pragma unroll
  for (int r = 0; r < 2; ++r) limit[r] = p.causal ? min(rows[r] + p.causal_off, p.Sk - 1) : p.Sk - 1;
  // documents: each row's limits narrowed to its document's keys (a row with none keeps its carried state)
  if constexpr (kDoc) {
#pragma unroll
    for (int r = 0; r < 2; ++r) limit[r] = min(limit[r], doc_hi[r] - 1);
  }
  const int limit_min = min(limit[0], limit[1]);
  // band: this group's tiles start at my0; keys below lo_limit[r] are masked for row r
  int my0 = 0, lo_limit[2] = {0, 0};
  if constexpr (kBand) {
    my0 = fwd_first_tile(row0 + wg * 64, p);
    lo_limit[0] = rows[0] + p.lo;
    lo_limit[1] = rows[1] + p.lo;
  }
  if constexpr (kDoc) {
    my0 = doc_first;
#pragma unroll
    for (int r = 0; r < 2; ++r) lo_limit[r] = max(lo_limit[r], doc_lo[r]);
  }
  const int lo_limit_max = max(lo_limit[0], lo_limit[1]);
  // ALiBi: slope in log2 units, and each row's reference distance (alibi_dref)
  float slope2 = 0.f;
  int64_t dref[2] = {0, 0};
  if constexpr (kAlibi) {
    slope2 = __ldg(p.slopes + (int64_t)b * p.slopes_sb + h) * kLog2e;
    dref[0] = alibi_dref(rows[0], p);
    dref[1] = alibi_dref(rows[1], p);
  }

  float o[kOReg];
  float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};  // l: this thread's partial row sums
#pragma unroll
  for (int i = 0; i < kOReg; ++i) o[i] = 0.f;
  if (p.load_state) {
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      if (rows[r] >= p.Sq) continue;
      const float lse_prev = p.lse[(int64_t)b * p.lse_sb + (int64_t)h * p.lse_sh + rows[r]];
      if (lse_prev != -INFINITY) {
        m[r] = lse_prev * kLog2e;
        if constexpr (kAlibi) {
          dref[r] = alibi_carried_ref(dref[r], m[r], slope2);
          m[r] += slope2 * (float)dref[r];
        }
        l[r] = t == 0 ? 1.f : 0.f;  // counted once per row
      }
      const float* src = p.o_acc + (int64_t)b * p.oacc_sb + (int64_t)rows[r] * p.oacc_ss + (int64_t)h * p.oacc_sh;
#pragma unroll
      for (int c = 0; c < kD / 8; ++c) {
        const float2 f = __ldg(reinterpret_cast<const float2*>(src + 8 * c + 2 * t));
        o[4 * c + 2 * r] = f.x;
        o[4 * c + 2 * r + 1] = f.y;
      }
    }
  }

  const uint32_t q_base = smem_u32(sQ) + wg * 64 * 128;  // this group's 64 rows inside every Q box
  mbar_wait(&bars->q_full, 0);
  for (int i = 0; i < n_tiles; ++i) {
    const int ks = i % kKStages, kph = (i / kKStages) & 1;
    const int vs = i % kVStages, vph = (i / kVStages) & 1;
    const bool work = kBand ? (t0 + i >= my0 && t0 + i < n_mine) : i < n_mine;  // warpgroup-uniform
    mbar_wait(&bars->k_full[ks], kph);
    float sc[64];
    if (work) {
      const uint32_t k_base = smem_u32(sK + ks * kTileBytes);
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < kD / 16; ++kk) {
        const uint32_t off = (kk >> 2) * kBoxBytes + (kk & 3) * 32;
        wgmma_ss_n128<kBF16, 0, 0>(sc, make_desc(q_base + off, 16, 1024), make_desc(k_base + off, 16, 1024),
                                   kk > 0 ? 1u : 0u);
      }
      wgmma_commit();
      wgmma_wait<0>();
      fence_regs<64>(sc);
      // scores in log2 units (+ key bias), masked keys -> -inf
      const int key0 = (t0 + i) * kBlockN;
      if constexpr (kBias) {
        mbar_wait(&bars->b_full[ks], kph);
        const float* bias = sBias + ks * kBlockN;
#pragma unroll
        for (int c = 0; c < 16; ++c) {
          const float2 bb = *reinterpret_cast<const float2*>(bias + 8 * c + 2 * t);
#pragma unroll
          for (int r = 0; r < 2; ++r) {
            sc[4 * c + 2 * r] = fmaf(sc[4 * c + 2 * r], scale_log2, bb.x);
            sc[4 * c + 2 * r + 1] = fmaf(sc[4 * c + 2 * r + 1], scale_log2, bb.y);
          }
        }
      } else if constexpr (kAlibi) {
        // d = pstride (a - c) + dist0 over this group's 64 rows x 128 keys; j = c - key0 (0..127)
        const int64_t base = (int64_t)p.pstride * (row0 + wg * 64 - key0) + p.dist0;
        const int64_t dmin = base - (int64_t)p.pstride * (kBlockN - 1), dmax = base + (int64_t)p.pstride * 63;
        const float pf = (float)p.pstride;
        if (dmin >= 0 || dmax <= 0) {
          // one sign s: |d| - dref = x_row - s pstride j, with the exact integer x_row = s (pstride (a - key0) +
          // dist0) - dref >= 0.  Score += -slope x_row (per row) + s slope pstride j (per key).
          const int sg = dmin >= 0 ? 1 : -1;
          float rowb[2];
#pragma unroll
          for (int r = 0; r < 2; ++r)
            rowb[r] = -slope2 * (float)(sg * ((int64_t)p.pstride * (rows[r] - key0) + p.dist0) - dref[r]);
          const float ks = sg > 0 ? slope2 * pf : -slope2 * pf, kt = ks * (float)(2 * t);
#pragma unroll
          for (int c = 0; c < 16; ++c)
#pragma unroll
            for (int e = 0; e < 4; ++e)
              sc[4 * c + e] = fmaf(sc[4 * c + e], scale_log2, rowb[e >> 1] + fmaf(ks, (float)(8 * c + (e & 1)), kt));
        } else {
          // the tile crosses d = 0, so every |d| here is below 256 pstride and exact in fp32
          float dr[2], dreff[2];
#pragma unroll
          for (int r = 0; r < 2; ++r) {
            dr[r] = (float)((int64_t)p.pstride * (rows[r] - key0 - 2 * t) + p.dist0);
            dreff[r] = slope2 * (float)dref[r];
          }
#pragma unroll
          for (int c = 0; c < 16; ++c)
#pragma unroll
            for (int e = 0; e < 4; ++e)
              sc[4 * c + e] = fmaf(-slope2, fabsf(fmaf(-pf, (float)(8 * c + (e & 1)), dr[e >> 1])),
                                   fmaf(sc[4 * c + e], scale_log2, dreff[e >> 1]));
        }
      } else {
#pragma unroll
        for (int j = 0; j < 64; ++j) sc[j] *= scale_log2;
      }
      if (key0 + kBlockN - 1 > limit_min) {
#pragma unroll
        for (int c = 0; c < 16; ++c)
#pragma unroll
          for (int e = 0; e < 4; ++e)
            if (key0 + 8 * c + 2 * t + (e & 1) > limit[e >> 1]) sc[4 * c + e] = -INFINITY;
      }
      if constexpr (kBand) {  // the band's lower edge; a row whose keys of this tile are all masked keeps m = -inf
        if (key0 < lo_limit_max) {
#pragma unroll
          for (int c = 0; c < 16; ++c)
#pragma unroll
            for (int e = 0; e < 4; ++e)
              if (key0 + 8 * c + 2 * t + (e & 1) < lo_limit[e >> 1]) sc[4 * c + e] = -INFINITY;
        }
      }
    }
    // K (and the bias row) of this stage are no longer read by this warp
    __syncwarp();
    if (lane == 0) mbar_arrive(&bars->k_empty[ks]);
    if (work) {
      uint32_t pa[32];
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        float mx = -INFINITY;
#pragma unroll
        for (int c = 0; c < 16; ++c) mx = fmaxf(mx, fmaxf(sc[4 * c + 2 * r], sc[4 * c + 2 * r + 1]));
        mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
        mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
        const float m_new = fmaxf(m[r], mx);
        const float f = (m[r] == -INFINITY) ? 0.f : ex2(m[r] - m_new);
        const float neg_m = (m_new == -INFINITY) ? 0.f : -m_new;
        m[r] = m_new;
        float sum = 0.f;
#pragma unroll
        for (int c = 0; c < 16; ++c) {
          const float p0 = ex2(sc[4 * c + 2 * r] + neg_m), p1 = ex2(sc[4 * c + 2 * r + 1] + neg_m);
          sc[4 * c + 2 * r] = p0;
          sc[4 * c + 2 * r + 1] = p1;
          sum += p0 + p1;
        }
        l[r] = l[r] * f + sum;
#pragma unroll
        for (int c = 0; c < kD / 8; ++c) {
          o[4 * c + 2 * r] *= f;
          o[4 * c + 2 * r + 1] *= f;
        }
      }
#pragma unroll
      for (int j = 0; j < 32; ++j) pa[j] = pack2<kBF16>(sc[2 * j], sc[2 * j + 1]);
      mbar_wait(&bars->v_full[vs], vph);
      const uint32_t v_base = smem_u32(sV + vs * kTileBytes);
      fence_regs<32>(pa);
      fence_regs<kOReg>(o);
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < kBlockN / 16; ++kk) {
        const uint64_t dv = make_desc(v_base + kk * 16 * 128, kBoxBytes, 1024);
        if constexpr (kD == 128) wgmma_rs_n128<kBF16, 1>(o, pa + 4 * kk, dv, 1u);
        else wgmma_rs_n64<kBF16, 1>(o, pa + 4 * kk, dv, 1u);
      }
      wgmma_commit();
      wgmma_wait<0>();
      fence_regs<kOReg>(o);
    } else {
      mbar_wait(&bars->v_full[vs], vph);  // keeps the arrivals below in phase with the other warpgroup
    }
    __syncwarp();
    if (lane == 0) mbar_arrive(&bars->v_empty[vs]);
  }

  // ---------------------------------------------------------- epilogue
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    float lr = l[r];
    lr += __shfl_xor_sync(0xffffffffu, lr, 1);
    lr += __shfl_xor_sync(0xffffffffu, lr, 2);
    const int row = rows[r];
    if (row >= p.Sq) continue;
    const float inv_l = lr > 0.f ? 1.f / lr : 0.f;
    if constexpr (kAlibi) {  // back from the row's reference to the absolute bias
      if (t == 0)
        p.lse[(int64_t)b * p.lse_sb + (int64_t)h * p.lse_sh + row] =
            lr > 0.f ? (m[r] + lg2(lr) - slope2 * (float)dref[r]) * kLn2 : -INFINITY;
    } else {
      if (t == 0) p.lse[(int64_t)b * p.lse_sb + (int64_t)h * p.lse_sh + row] = lr > 0.f ? (m[r] + lg2(lr)) * kLn2 : -INFINITY;
    }
    if (p.store_lowp) {
      uint16_t* dst = reinterpret_cast<uint16_t*>(p.o_out) + (int64_t)b * p.oout_sb + (int64_t)row * p.oout_ss +
                      (int64_t)h * p.oout_sh + 2 * t;
#pragma unroll
      for (int c = 0; c < kD / 8; ++c)
        *reinterpret_cast<uint32_t*>(dst + 8 * c) = pack2<kBF16>(o[4 * c + 2 * r] * inv_l, o[4 * c + 2 * r + 1] * inv_l);
    } else {
      float* dst = p.o_acc + (int64_t)b * p.oacc_sb + (int64_t)row * p.oacc_ss + (int64_t)h * p.oacc_sh + 2 * t;
#pragma unroll
      for (int c = 0; c < kD / 8; ++c)
        *reinterpret_cast<float2*>(dst + 8 * c) = make_float2(o[4 * c + 2 * r] * inv_l, o[4 * c + 2 * r + 1] * inv_l);
    }
  }
}

template <bool kBF16, int kD, bool kBias, bool kBand>
__global__ void __launch_bounds__(kFwdThreads, 1)
fwd_chunk_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                 const __grid_constant__ CUtensorMap tmV, const FwdParams p) {
  fwd_chunk_body<kBF16, kD, kBias, kBand, false>(tmQ, tmK, tmV, p);
}

// ALiBi instantiations: fwd_alibi_sm90.cu
template <bool kBF16, int kD, bool kBand>
__global__ void __launch_bounds__(kFwdThreads, 1)
fwd_alibi_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                 const __grid_constant__ CUtensorMap tmV, const FwdParams p) {
  fwd_chunk_body<kBF16, kD, false, kBand, true>(tmQ, tmK, tmV, p);
}

// document instantiations: fwd_doc_sm90.cu
template <bool kBF16, int kD>
__global__ void __launch_bounds__(kFwdThreads, 1)
fwd_doc_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
               const __grid_constant__ CUtensorMap tmV, const FwdParams p) {
  fwd_chunk_body<kBF16, kD, false, true, false, true>(tmQ, tmK, tmV, p);
}

// Each tile TU instantiates its own kernels and hands fwd_chunk_run (fwd_sm90.cu), which launches every one of them,
// the kernel of a call's (dtype, head dim, ...).
using FwdKernel = void (*)(CUtensorMap, CUtensorMap, CUtensorMap, FwdParams);

// fwd_chunk_kernel of (dtype, head dim, bias) for this TU's kBand: fwd_sm90.cu kBand = false, fwd_band_sm90.cu true
template <bool kBand>
inline FwdKernel fwd_chunk_kernel_of(bool bf16, int D, bool bias) {
  if (bias)
    return D == 64 ? (bf16 ? fwd_chunk_kernel<true, 64, true, kBand> : fwd_chunk_kernel<false, 64, true, kBand>)
                   : (bf16 ? fwd_chunk_kernel<true, 128, true, kBand> : fwd_chunk_kernel<false, 128, true, kBand>);
  return D == 64 ? (bf16 ? fwd_chunk_kernel<true, 64, false, kBand> : fwd_chunk_kernel<false, 64, false, kBand>)
                 : (bf16 ? fwd_chunk_kernel<true, 128, false, kBand> : fwd_chunk_kernel<false, 128, false, kBand>);
}

FwdKernel fwd_band_kernel_of(bool bf16, int D, bool bias);   // fwd_band_sm90.cu
FwdKernel fwd_alibi_kernel_of(bool bf16, int D, bool band);  // fwd_alibi_sm90.cu
FwdKernel fwd_doc_kernel_of(bool bf16, int D);               // fwd_doc_sm90.cu

}  // namespace ba
