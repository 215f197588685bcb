// ba_bwd_chunk: one ring round of the backward on sm_90a.
//
// Replaces the reference's per-round flash_attn_2_cuda.bwd call
// (burst_utils.py:180-249; Triton twin lao.py:295-595) AND the three full-tensor
// "dq += buf; dk += buf; dv += buf" passes of burst_attn_interface.py:379-390:
// the kernel accumulates straight into fp32 dQ / dK / dV accumulators.
// delta = rowsum(O*dO) and the final lse are inputs (they travel with the
// Q-bundle), so O itself is never read here.
//
// One CTA owns one 128-key block of the home K/V chunk for one (batch, K/V head) and loops over the G query heads
// that share that K/V head (grouped-query attention; G = 1 for MHA) and, for each, over the 64-row blocks of the
// visiting Q-bundle: G x n_it steps, one pipeline whose stages and mbarrier phases run on across heads.
// Warpgroup 0 is the TMA producer (K, V once; Q, dO and the row statistics per step, 3 stages); warpgroups 1 and 2
// own 64 keys each and keep their dK, dV accumulators in registers across all G heads, so the epilogue does a
// single read-modify-write of dk_acc / dv_acc per CTA (no atomics; dK / dV stay deterministic):
//   S^T  = K_w Q_i^T,  dP^T = V_w dO_i^T      (wgmma SS m64n64, K-major operands)
//   P^T  = exp2(S^T c [+ bias] - lse2),  dS^T = P^T o (dP^T - delta)     (registers, thread = 2 key rows)
//   dS^T -> smem (double-buffered)
//   dV_w += P^T dO_i   (wgmma RS: P^T re-packed to 16 bit as the A operand, dO read MN-major)
//   dK_w += dS^T Q_i   (wgmma SS: the warpgroup's rows of the dS^T tile read K-major, Q read MN-major)
//   dQ_i = dS K        (wgmma SS, both operands MN-major; head dim 128: each warpgroup computes 64 of the dQ
//                       columns, head dim 64: warpgroup 1 alone) -> smem -> cp.reduce.async.bulk.tensor (fp32 add
//                       in L2) into dq_acc.
// A consumer warpgroup keeps its own MMAs running under its element-wise work, and across steps: the next step's
// S^T is issued between this step's dQ and dK, so the tensor cores have S^T and dK queued under the dQ staging, and
// dK and the next dP^T under the next P^T (five commit groups per step; four, without dQ, for the non-reducing
// warpgroup at head dim 64):
//   prologue: issue S^T_0 | empty group (stands for dK_{-1}) | issue dP^T_0
//   step j:   wait<2> (S^T_j done) | P^T (exp2, bias, masks) + pack, under dK_{j-1} and dP^T_j | wait<0> | release
//             the Q / dO stage of step j-1 | issue dV | dS^T + pack + store to smem, under dV | barrier with the
//             other warpgroup | issue dQ | issue S^T_{j+1} | issue dK | wait<2> (dV, dQ done) | stage dQ +
//             reduce-add, under S^T_{j+1} and dK | issue dP^T_{j+1}
//   the last step issues nothing for a next one and ends with wait<0> and the release of its stage.
// The operands of an MMA (packed P^T for dV, the dS^T tile for dQ and dK) stay untouched until the wait that retires
// its group.
// smem (D = 128): K 32K, V 32K, Q 3x16K, dO 3x16K, dS^T 2x16K, dQ staging 16K per reducing warpgroup (single-
// buffered: its next write waits for the previous reduce to have read it), row statistics 1.5K.
// The dQ staging of a warpgroup is two [64 rows][32 fp32] SW128 boxes, one reduce-add each; lanes with odd row
// index store their 8-column chunks in a permuted order, so every STS.64 of the staging is conflict-free (2
// wavefronts; the bank arithmetic is next to the stores).
//
// Band mask (kBand, sliding-window attention): key c is visible to row a iff a + lo <= c (and c <= a + causal_off
// when causal).  A key block then visits the Q blocks [i_begin, i_end) only, and P^T gets the band's lower edge.
// kBand = false is the kernel without a lower edge (bwd_sm90.cu); kBand = true lives in bwd_band_sm90.cu.
//
// ALiBi (kAlibi, bwd_alibi_kernel in bwd_alibi_sm90.cu): P^T gets -slope |pstride (q - c) + dist0| (see bwd_chunk_body).
//
// Packed documents (kDoc, bwd_doc_kernel in bwd_doc_sm90.cu; always with kBand): a key block visits only the Q blocks
// of the documents of its first and last key, the loader stages each Q row's document keys relative to the block
// (two int16 in [0, 128]) with the row statistics and flags a Q block whose rows do not all see the whole key block,
// and P^T gets the per-element document mask on flagged tiles only.
#pragma once
#include <math.h>
#include <stdlib.h>

#include <type_traits>

#include "doc_sm90.cuh"
#include "host_common.h"
#include "sm90_ptx.cuh"

namespace ba {

constexpr int kBwdThreads = 384;  // warpgroup 0: loader (warp 0); warpgroups 1, 2: MMA + element-wise
constexpr int kBwdN = 128;        // keys per CTA
constexpr int kBwdM = 64;         // query rows per block of the Q-bundle
// Q / dO / statistics stages.  A stage is released at the top of the step after the one that read it, and the
// next step's stage is needed in the middle of a step, so with 3 stages the loader has about 1.5 steps per load.
constexpr int kBwdStages = 3;

struct BwdParams {
  const float* lse;
  int64_t lse_sb, lse_sh;
  const float* delta;
  int64_t dl_sb, dl_sh;
  float* dk_acc;
  int64_t dk_sb, dk_ss, dk_sh;
  float* dv_acc;
  int64_t dv_sb, dv_ss, dv_sh;
  int B, Sq, Sk, H;
  int G;  // query heads per K/V head (grouped-query attention; 1 = MHA): K/V head hk serves heads hk*G .. hk*G+G-1
  float scale, scale_log2;
  int causal, causal_off;
  const float* bias;  // optional additive bias per key [B|1, H, Sk] (fp32, indexed by the query head), or null
  int64_t bias_sb, bias_sh;
  int* sem;     // deterministic mode: [B][H][nQ] turn counters ordering the dQ reductions by key block; else null
  int* ticket;  // deterministic mode: [B][H/G] key-block tickets (a CTA's key block = the order in which it STARTED)
  int lo;       // kBand: key c is visible to row a only if c >= a + lo
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

// ALiBi over the tile of the 64 rows from q0 and the 128 keys from k0: +1 or -1 when d has that sign (or is 0) on
// the whole tile, 0 when the tile crosses d = 0
__device__ __forceinline__ int alibi_tile_sign(int q0, int k0, const BwdParams& p) {
  const int64_t base = (int64_t)p.pstride * (q0 - k0) + p.dist0;
  if (base - (int64_t)p.pstride * (kBwdN - 1) >= 0) return 1;
  if (base + (int64_t)p.pstride * (kBwdM - 1) <= 0) return -1;
  return 0;
}

__device__ __forceinline__ int ld_acquire_gpu(const int* p) {
  int v;
  asm volatile("ld.acquire.gpu.global.s32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_release_gpu(int* p, int v) {
  asm volatile("st.release.gpu.global.s32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}

struct __align__(8) BwdBarriers {
  uint64_t kv_full;
  uint64_t q_full[kBwdStages], q_empty[kBwdStages];  // Q, dO and the row statistics of one Q block
  int key_block;                                     // deterministic mode: this CTA's ticket
};
static_assert(sizeof(BwdBarriers) <= 64, "BwdLayout reserves 64 bytes for the barriers");

// smem carve-up (bytes from the 1 KiB-aligned base); head dim kD (64 or 128)
template <int kD>
struct BwdLayout {
  static_assert(kD == 64 || kD == 128, "head dim 64 or 128");
  static constexpr int kBoxes = kD / 64;
  static constexpr int kBoxKV = kBwdN * 128;  // 16 KiB: [128 keys][64 cols] SW128 box
  static constexpr int kBoxQ = kBwdM * 128;   // 8 KiB: [64 rows][64 cols] SW128 box
  static constexpr int kBoxDQ = kBwdM * 128;  // 8 KiB: [64 rows][32 fp32 cols] SW128 box
  static constexpr int kOffK = 0;
  static constexpr int kOffV = kOffK + kBoxes * kBoxKV;
  static constexpr int kOffQ = kOffV + kBoxes * kBoxKV;                // kBwdStages stages
  static constexpr int kOffDO = kOffQ + kBwdStages * kBoxes * kBoxQ;   // kBwdStages stages
  static constexpr int kOffDS = kOffDO + kBwdStages * kBoxes * kBoxQ;  // 2 x [128 keys][64 q] SW128
  static constexpr int kOffDQ = kOffDS + 2 * kBwdN * 128;              // per reducing warpgroup 2 dQ boxes (64 columns)
  static constexpr int kOffStat = kOffDQ + kBoxes * 2 * kBoxDQ;  // kBwdStages stages x [lse2 | delta] x 64 fp32
  static constexpr int kOffBar = kOffStat + kBwdStages * 2 * kBwdM * 4;
  static constexpr int kSmemBytes = kOffBar + 64;  // no align slack: the dynamic smem base is checked to be 1 KiB aligned
  static_assert(kSmemBytes <= 232448, "backward kernel exceeds 227 KiB of shared memory");
  static_assert(kOffDQ % 1024 == 0, "SW128 dQ staging boxes need 1 KiB alignment");
  // kDoc only, past the end of the other kernels' carve-up: per stage, each Q row's document keys relative to the
  // key block as two int16 [lo | hi << 16], and the stage's "crosses a document edge" flag (padded to 16 bytes)
  static constexpr int kDocStageB = kBwdM * 4 + 16;
  static constexpr int kOffDoc = kSmemBytes;
  static constexpr int kSmemDocBytes = kOffDoc + kBwdStages * kDocStageB;
  static_assert(kSmemDocBytes <= 232448, "backward document kernel exceeds 227 KiB of shared memory");
};

// The kernel body; bwd_chunk_kernel (kAlibi = false) and bwd_alibi_kernel (kAlibi = true, no key bias) wrap it.
// ALiBi: on a tile where d has one sign s, -slope |d| = -slope s (pstride (q - k0) + dist0) + s slope pstride (c - k0):
// the loader folds the per-row term into the row's lse2 (it is per tile: k0 is the CTA's), and the per-key term sits
// where the key bias goes.  On a tile that crosses d = 0, every |d| is below 192 pstride, exact in fp32, and the bias
// is formed per element.
template <bool kBF16, int kD, bool kBand, bool kAlibi, bool kDoc = false>
__device__ __forceinline__ void bwd_chunk_body(const CUtensorMap& tmQ, const CUtensorMap& tmK, const CUtensorMap& tmV,
                                               const CUtensorMap& tmDO, const CUtensorMap& tmDQ, const BwdParams& p) {
  static_assert(!kDoc || (kBand && !kAlibi), "documents run on the band path, without ALiBi");
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = smem_raw;
  if ((smem_u32(smem) & 1023u) != 0) __trap();  // SWIZZLE_128B atoms need a 1 KiB-aligned base
  using L = BwdLayout<kD>;
  constexpr int kBoxes = L::kBoxes, kBoxKV = L::kBoxKV, kBoxQ = L::kBoxQ, kDQBox = L::kBoxDQ, kAcc = kD / 2;
  constexpr int kQStageB = kBoxes * kBoxQ;
  float* sStat = reinterpret_cast<float*>(smem + L::kOffStat);
  BwdBarriers* bars = reinterpret_cast<BwdBarriers*>(smem + L::kOffBar);

  const int warp = __shfl_sync(0xffffffffu, threadIdx.x >> 5, 0);
  const int lane = threadIdx.x & 31;
  const int hk = blockIdx.y, b = blockIdx.z;  // K/V head; its query heads are h0 .. h0 + G - 1
  const int h0 = hk * p.G;
  // Key block of this CTA.  Deterministic mode orders the dQ reductions by key block and makes a CTA wait for
  // all lower key blocks; to make that wait deadlock-free without assuming anything about the order in which
  // the hardware dispatches blockIdx.x, the key block is a ticket drawn when the CTA starts: every lower
  // ticket then belongs to a CTA that is already resident.  Tickets are per (batch, K/V head): the CTAs that
  // share one are exactly the ones whose dQ reductions meet on the same (query head, Q block) turn counters.
  int kb = blockIdx.x;
  if (p.sem) {
    if (threadIdx.x == 0) bars->key_block = atomicAdd(p.ticket + b * (p.H / p.G) + hk, 1);
    __syncthreads();
    kb = bars->key_block;
  }
  const int k0 = kb * kBwdN;
  const int nQ = (p.Sq + kBwdM - 1) / kBwdM;
  // first Q block that can see any key of this block: q >= k0 - off (the same for every query head of the group)
  int i_begin = p.causal ? max(0, k0 - p.causal_off) / kBwdM : 0;
  // band: one past the last Q block that can see any key of this block: q + lo <= min(k0 + 127, Sk - 1)
  int i_end = nQ;
  if constexpr (kBand) {
    const int q_last = min(k0 + kBwdN - 1, p.Sk - 1) - p.lo;
    i_end = q_last < 0 ? 0 : min(nQ, q_last / kBwdM + 1);
  }
  // documents: only the rows of the documents of the block's first and last key (documents never decrease along
  // the keys, so these two bound the rows of every key in between)
  if constexpr (kDoc) {
    int r_lo, r_hi, unused;
    doc_interval(p.k_pos0 + p.pstride * k0, p.cu, p.n_docs, p.q_pos0, p.pstride, p.Sq, &r_lo, &unused);
    doc_interval(p.k_pos0 + p.pstride * min(k0 + kBwdN - 1, p.Sk - 1), p.cu, p.n_docs, p.q_pos0, p.pstride,
                 p.Sq, &unused, &r_hi);
    i_begin = max(i_begin, r_lo / kBwdM);
    i_end = min(i_end, (r_hi + kBwdM - 1) / kBwdM);
  }
  const int n_it = max(0, i_end - i_begin);
  if (n_it == 0) return;  // nothing visible: dK/dV contributions are zero (uniform exit, no barriers yet)
  const int n_steps = p.G * n_it;  // step j: query head h0 + j / n_it, Q block i_begin + j % n_it

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmQ);
    tma_prefetch_desc(&tmK);
    tma_prefetch_desc(&tmV);
    tma_prefetch_desc(&tmDO);
    tma_prefetch_desc(&tmDQ);
    mbar_init(&bars->kv_full, 1);
    for (int s = 0; s < kBwdStages; ++s) {
      mbar_init(&bars->q_full[s], 1);
      mbar_init(&bars->q_empty[s], 8);  // one elected arrive per consumer warp
    }
    fence_mbar_init();
  }
  __syncthreads();

  if (warp < 4) {
    // ============================================================ loader (warp 0)
    reg_alloc_dec<24>();
    if (warp != 0) return;
    if (lane == 0) {
      mbar_arrive_expect_tx(&bars->kv_full, 2 * kBoxes * kBoxKV);
      for (int half = 0; half < kBoxes; ++half) {
        tma_load_4d(smem + L::kOffK + half * kBoxKV, &tmK, &bars->kv_full, half * 64, hk, k0, b);
        tma_load_4d(smem + L::kOffV + half * kBoxKV, &tmV, &bars->kv_full, half * 64, hk, k0, b);
      }
    }
    int it = 0, h = h0;  // Q block (relative to i_begin) and query head of this step
    int st = 0, ph = 0;  // stage of this step (step % kBwdStages) and its phase ((step / kBwdStages) & 1)
    for (int step = 0; step < n_steps; ++step) {
      const int q0 = (i_begin + it) * kBwdM;
      [[maybe_unused]] float slope2 = 0.f;
      [[maybe_unused]] int sg = 0;
      if constexpr (kAlibi) {
        slope2 = __ldg(p.slopes + (int64_t)b * p.slopes_sb + h) * kLog2e;
        sg = alibi_tile_sign(q0, k0, p);
      }
      mbar_wait(&bars->q_empty[st], ph ^ 1);
      // row statistics of this Q block (lane handles rows lane, lane + 32): lse in log2 units, delta
      float* stat = sStat + st * 2 * kBwdM;
#pragma unroll
      for (int j = 0; j < 2; ++j) {
        const int row = q0 + lane + 32 * j;
        float l = INFINITY, dl = 0.f;  // +inf: padding row, or a row that saw no key at all -> P = 0
        if (row < p.Sq) {
          l = __ldg(p.lse + (int64_t)b * p.lse_sb + (int64_t)h * p.lse_sh + row);
          dl = __ldg(p.delta + (int64_t)b * p.dl_sb + (int64_t)h * p.dl_sh + row);
          if (l == -INFINITY) l = INFINITY;
        }
        if constexpr (kAlibi) {  // + slope s (pstride (q - k0) + dist0), the exact integer converted once
          const float x = (float)(sg * ((int64_t)p.pstride * (row - k0) + p.dist0));
          stat[lane + 32 * j] = fmaf(slope2, x, l * kLog2e);
        } else {
          stat[lane + 32 * j] = l * kLog2e;
        }
        stat[kBwdM + lane + 32 * j] = dl;
      }
      if constexpr (kDoc) {  // each row's document keys relative to k0, and whether any row misses a key of the block
        uint32_t* dw = reinterpret_cast<uint32_t*>(smem + L::kOffDoc + st * L::kDocStageB);
        bool cross = false;
#pragma unroll 1
        for (int j = 0; j < 2; ++j) {
          const int row = q0 + lane + 32 * j;
          int lo = 0, hi = 0;  // padding row: no key (its P is 0 anyway)
          if (row < p.Sq) {
            doc_interval(p.q_pos0 + p.pstride * row, p.cu, p.n_docs, p.k_pos0, p.pstride, p.Sk, &lo, &hi);
            lo = min(max(lo - k0, 0), kBwdN);
            hi = min(max(hi - k0, 0), kBwdN);
            cross |= lo > 0 || hi < min(kBwdN, p.Sk - k0);
          }
          dw[lane + 32 * j] = (uint32_t)lo | ((uint32_t)hi << 16);
        }
        const unsigned any = __ballot_sync(0xffffffffu, cross);
        if (lane == 0) dw[kBwdM] = any != 0u;
      }
      __syncwarp();
      if (lane == 0) {
        mbar_arrive_expect_tx(&bars->q_full[st], 2 * kQStageB);
        for (int half = 0; half < kBoxes; ++half) {
          tma_load_4d(smem + L::kOffQ + st * kQStageB + half * kBoxQ, &tmQ, &bars->q_full[st], half * 64, h, q0, b);
          tma_load_4d(smem + L::kOffDO + st * kQStageB + half * kBoxQ, &tmDO, &bars->q_full[st], half * 64, h, q0, b);
        }
      }
      __syncwarp();
      if (++it == n_it) it = 0, ++h;
      if (++st == kBwdStages) st = 0, ph ^= 1;
    }
    return;
  }

  // ============================================================ consumers (64 keys per warpgroup)
  reg_alloc_inc<240>();
  const int wg = (threadIdx.x >> 7) - 1;
  const int tid = threadIdx.x & 127;
  const int w = warp & 3, g = lane >> 2, t = lane & 3;
  const int kr_lo = wg * 64 + 16 * w + g;  // this thread's key rows within the block: kr_lo, kr_lo + 8
  const int keys[2] = {k0 + kr_lo, k0 + kr_lo + 8};
  const float scale_log2 = p.scale_log2;
  // additive bias of this thread's keys, in log2 units (scores = q k^T scale + bias[key]; reference lao.py:155-173,
  // "vector" bias): a per-row scalar in this key-row layout, folded into the exponent's FMA; the bias is per query
  // head, so it is (re)loaded at the first step of every head
  float bias2[2];
  const int n_red = kD == 128 ? 2 : 1;

  float dk[kAcc], dv[kAcc];
#pragma unroll
  for (int i = 0; i < kAcc; ++i) dk[i] = dv[i] = 0.f;
  // the zeros are set here, not sunk under the first MMAs (writing an accumulator register while a wgmma group is in
  // flight makes ptxas serialize every wgmma of the kernel)
  fence_regs<kAcc>(dk);
  fence_regs<kAcc>(dv);

  const uint32_t sK = smem_u32(smem + L::kOffK), sV = smem_u32(smem + L::kOffV);
  const uint32_t kw = wg * 64 * 128;  // this group's 64 key rows inside every K / V box
  uint8_t* sDQ = smem + L::kOffDQ + wg * 2 * kDQBox;
  auto q_stage = [&](int st) { return smem_u32(smem + L::kOffQ + st * kQStageB); };
  auto do_stage = [&](int st) { return smem_u32(smem + L::kOffDO + st * kQStageB); };
  // acc = X_w Y^T as one commit group (wgmma SS m64n64, K-major operands): S^T = K_w Q^T or dP^T = V_w dO^T
  auto issue_xt = [&](float* acc, uint32_t sX, uint32_t sY) {
    // the descriptors are rebuilt at each issue: hoisted out of the step loop, the K ones would hold 16 registers
    // for the whole step, and the step would spill
    asm volatile("" : "+r"(sX));
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < kD / 16; ++kk) {
      const uint32_t okv = (kk >> 2) * kBoxKV + kw + (kk & 3) * 32, oq = (kk >> 2) * kBoxQ + (kk & 3) * 32;
      wgmma_ss_n64<kBF16, 0, 0>(acc, make_desc(sX + okv, 16, 1024), make_desc(sY + oq, 16, 1024), kk > 0 ? 1u : 0u);
    }
    wgmma_commit();
  };
  mbar_wait(&bars->kv_full, 0);

  // The steps of one consumer warpgroup.  kRed: it owns 64 columns of dQ (both warpgroups at head dim 128,
  // warpgroup 1 alone at head dim 64).  dK of a step is retired in the next one, so the role is fixed for the whole
  // loop rather than branched on per step: each wgmma group is issued and waited for on one path (a group across a
  // divergent path makes ptxas serialize every wgmma of the kernel).
  auto consume = [&](auto red) {
    constexpr bool kRed = decltype(red)::value;
    float s[32], dp[32];  // S^T (P^T in place) and dP^T of this step: issued by the step before
    int it = 0, h = h0;   // Q block (relative to i_begin) and query head of this step
    int st = 0, ph = 0;   // Q / dO / statistics stage of this step and its q_full phase
    mbar_wait(&bars->q_full[0], 0);
    issue_xt(s, sK, q_stage(0));
    wgmma_commit();  // an empty group in the place of the previous step's dK, so that every step waits alike
    issue_xt(dp, sV, do_stage(0));

    // One step; kNext (every step but the last): issue the next step's S^T and dP^T.  The last step is a copy of
    // its own, so that no wgmma is issued under a runtime condition.
    auto step_body = [&](auto next, int step) {
      constexpr bool kNext = decltype(next)::value;
      const int q0 = (i_begin + it) * kBwdM;
      const uint32_t sQ = q_stage(st), sDO = do_stage(st);
      const float* stat = sStat + st * 2 * kBwdM;
      [[maybe_unused]] const uint32_t* dw = nullptr;  // documents: this stage's row intervals, flag at [kBwdM]
      [[maybe_unused]] bool need_doc = false;
      if constexpr (kDoc) {
        dw = reinterpret_cast<const uint32_t*>(smem + L::kOffDoc + st * L::kDocStageB);
        need_doc = dw[kBwdM] != 0u;
      }
      // ALiBi: the bias relative to the row term the loader folded into lse2 is ma |ka[r] + kc (q - q0)|.  One-sign
      // tile s: ma = s slope, ka = pstride (c - k0), kc = 0.  Crossing tile: ma = -slope, ka + kc (q - q0) = d, with
      // ka = pstride (q0 + 2 t - c) + dist0 (small: the 32-bit sum wraps, and its true value fits) and kc = pstride.
      [[maybe_unused]] float ma = 0.f, kc = 0.f, ka[2];
      if constexpr (kAlibi) {
        const float slope2 = __ldg(p.slopes + (int64_t)b * p.slopes_sb + h) * kLog2e;
        const int sg = alibi_tile_sign(q0, k0, p);
        ma = sg > 0 ? slope2 : -slope2;
        kc = sg == 0 ? (float)p.pstride : 0.f;
#pragma unroll
        for (int r = 0; r < 2; ++r)
          ka[r] = sg == 0 ? (float)(int)((unsigned)p.pstride * (unsigned)(q0 + 2 * t - keys[r]) + (unsigned)p.dist0)
                          : (float)(p.pstride * (keys[r] - k0));
      } else if (it == 0) {
#pragma unroll
        for (int r = 0; r < 2; ++r)
          bias2[r] = (p.bias && keys[r] < p.Sk)
                         ? __ldg(p.bias + (int64_t)b * p.bias_sb + (int64_t)h * p.bias_sh + keys[r]) * kLog2e
                         : 0.f;
      }
      // in flight, oldest first: S^T, dK of the previous step, dP^T; P^T is computed from S^T while the other two run
      wgmma_wait<2>();  // S^T done
      fence_regs<32>(s);

      // P^T in place of S^T (fp32, kept for dS^T) and packed to 16 bit as the A operand of dV.
      // visible iff key <= q + off  <=>  q >= key - off ; whole block visible when q0 + off >= k0 + 127
      const bool need_mask = p.causal && (q0 + p.causal_off < k0 + kBwdN - 1);
      // band: visible only if key >= q + lo; the whole block passes when k0 >= q0 + 63 + lo
      const bool need_lo = kBand && (q0 + kBwdM - 1 + p.lo > k0);
      uint32_t pp[16];
#pragma unroll
      for (int c = 0; c < 8; ++c) {
        const float2 l2 = *reinterpret_cast<const float2*>(stat + 8 * c + 2 * t);
#pragma unroll
        for (int r = 0; r < 2; ++r) {
          const int e = 4 * c + 2 * r;
          float p0, p1;
          if constexpr (kAlibi) {
            const float x0 = fmaf(ma, fabsf(fmaf(kc, (float)(8 * c), ka[r])), -l2.x);
            const float x1 = fmaf(ma, fabsf(fmaf(kc, (float)(8 * c + 1), ka[r])), -l2.y);
            p0 = ex2(fmaf(s[e], scale_log2, x0));
            p1 = ex2(fmaf(s[e + 1], scale_log2, x1));
          } else {
            p0 = ex2(fmaf(s[e], scale_log2, bias2[r] - l2.x));
            p1 = ex2(fmaf(s[e + 1], scale_log2, bias2[r] - l2.y));
          }
          if (keys[r] >= p.Sk) p0 = p1 = 0.f;
          if (need_mask) {
            const int q = q0 + 8 * c + 2 * t;
            if (q < keys[r] - p.causal_off) p0 = 0.f;
            if (q + 1 < keys[r] - p.causal_off) p1 = 0.f;
          }
          if (need_lo) {  // false at compile time without kBand
            const int q = q0 + 8 * c + 2 * t;
            if (q + p.lo > keys[r]) p0 = 0.f;
            if (q + 1 + p.lo > keys[r]) p1 = 0.f;
          }
          if constexpr (kDoc) {
            if (need_doc) {  // key row kr of row q is visible iff lo(q) <= kr < hi(q)
              const uint2 iv = *reinterpret_cast<const uint2*>(dw + 8 * c + 2 * t);
              const uint32_t kr = (uint32_t)(keys[r] - k0);
              if (kr < (iv.x & 0xffffu) || kr >= (iv.x >> 16)) p0 = 0.f;
              if (kr < (iv.y & 0xffffu) || kr >= (iv.y >> 16)) p1 = 0.f;
            }
          }
          s[e] = p0, s[e + 1] = p1;
          pp[2 * c + r] = pack2<kBF16>(p0, p1);
        }
      }

      // dV += P^T dO   (B operand: [q rows][d] tile read MN-major); pp is read by the MMA until the wait<1> below
      wgmma_wait<0>();  // dK of the previous step and dP^T done
      fence_regs<32>(dp);
      fence_regs<16>(pp);
      fence_regs<kAcc>(dv);
      fence_regs<kAcc>(dk);
      if (step > 0) {
        // dK of the previous step was the last reader of that step's Q, dO and statistics
        __syncwarp();
        if (lane == 0) mbar_arrive(&bars->q_empty[st == 0 ? kBwdStages - 1 : st - 1]);
      }
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < kBwdM / 16; ++kk) {
        const uint64_t d_do = make_desc(sDO + kk * 16 * 128, kBoxQ, 1024);
        if constexpr (kD == 128) wgmma_rs_n128<kBF16, 1>(dv, pp + 4 * kk, d_do, 1u);
        else wgmma_rs_n64<kBF16, 1>(dv, pp + 4 * kk, d_do, 1u);
      }
      wgmma_commit();

      // dS^T = P^T o (dP^T - delta) while dV runs
      uint32_t ds[16];
#pragma unroll
      for (int c = 0; c < 8; ++c) {
        const float2 dl = *reinterpret_cast<const float2*>(stat + kBwdM + 8 * c + 2 * t);
#pragma unroll
        for (int r = 0; r < 2; ++r) {
          const int e = 4 * c + 2 * r;
          ds[2 * c + r] = pack2<kBF16>(s[e] * (dp[e] - dl.x), s[e + 1] * (dp[e + 1] - dl.y));
        }
      }

      // dS^T -> smem [128 keys][64 q] (SW128: 16-byte chunk j of row r at j ^ (r % 8)), double-buffered by step
      // parity: the buffer written here was last read by the dQ and dK MMAs of step - 2.  Each reducing warpgroup's
      // wgmma_wait<1> of step - 2 completes its dQ group (dV and dQ are the two oldest of its three groups), and that
      // wait comes before the warpgroup reaches the barrier of step - 1, which this warpgroup has passed.  dK reads
      // only this warpgroup's own 64 key rows, and its group was retired by this warpgroup's first wait of step - 1.
      uint8_t* sDS = smem + L::kOffDS + (step & 1) * kBwdN * 128;
#pragma unroll
      for (int c = 0; c < 8; ++c)
#pragma unroll
        for (int r = 0; r < 2; ++r) {
          const int kr = kr_lo + 8 * r;
          *reinterpret_cast<uint32_t*>(sDS + kr * 128 + ((c ^ (kr & 7)) << 4) + 4 * t) = ds[2 * c + r];
        }
      fence_proxy_async_smem();
      named_bar_sync(1, 256);

      // dQ[:, 64 wg .. 64 wg + 63] = dS K  (A = dS^T tile read MN-major, B = K tile read MN-major), then the next
      // step's S^T, then dK += dS^T Q (A = this warpgroup's 64 rows of the dS^T tile read K-major, B = Q read
      // MN-major).  Groups complete in issue order, so with S^T ahead of dK the next step's first wait retires S^T
      // alone: dK and the next dP^T stay queued under the next P^T, and S^T and dK under the dQ staging below.
      // dK reads dS^T from smem rather than as packed registers: those 16 registers would stay live through the
      // staging, beside dq and the next S^T, and the staging would exceed the register budget.
      // The next step's stage is step - 2's, which both warpgroups released in step - 1, before its barrier, so
      // the loader can fill it and the wait ends.
      const int st_next = st == kBwdStages - 1 ? 0 : st + 1;
      const int ph_next = st_next == 0 ? ph ^ 1 : ph;
      [[maybe_unused]] float dq[32];
      fence_regs<kAcc>(dk);
      wgmma_fence();
      if constexpr (kRed) {
        const uint32_t a0 = smem_u32(sDS), b0 = sK + wg * kBoxKV;
#pragma unroll
        for (int kk = 0; kk < kBwdN / 16; ++kk)
          wgmma_ss_n64<kBF16, 1, 1>(dq, make_desc(a0 + kk * 16 * 128, 8192, 1024),
                                    make_desc(b0 + kk * 16 * 128, kBoxKV, 1024), kk > 0 ? 1u : 0u);
        wgmma_commit();
      }
      if constexpr (kNext) {
        mbar_wait(&bars->q_full[st_next], ph_next);
        fence_regs<32>(s);
        issue_xt(s, sK, q_stage(st_next));
      }
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < kBwdM / 16; ++kk) {
        const uint64_t d_ds = make_desc(smem_u32(sDS) + kw + kk * 32, 16, 1024);
        const uint64_t d_q = make_desc(sQ + kk * 16 * 128, kBoxQ, 1024);
        if constexpr (kD == 128) wgmma_ss_n128<kBF16, 0, 1>(dk, d_ds, d_q, 1u);
        else wgmma_ss_n64<kBF16, 0, 1>(dk, d_ds, d_q, 1u);
      }
      wgmma_commit();
      // dV and dQ done; the next S^T (if any) and dK may still run
      if constexpr (kNext) wgmma_wait<2>();
      else wgmma_wait<1>();
      fence_regs<kAcc>(dv);
      fence_regs<16>(pp);
      // dP^T follows the staging: issued before it, its 32 accumulators would be live beside dq and push the
      // staging over the register budget.

      if constexpr (kRed) {
        fence_regs<32>(dq);
        const uint32_t bar_id = 2 + wg;
        if (tid == 0) tma_store_wait_read<0>();  // the previous reduce has finished reading the staging tile
        named_bar_sync(bar_id, 128);
        // This thread holds dQ rows 16 w + g + 8 r (row % 8 = g) at columns 8 c + 2 t, 8 c + 2 t + 1.  Column
        // 8 c + 2 t lies in box c / 4, 16-byte chunk j = 2 (c % 4) + t / 2 of its row, at byte 8 (t % 2) of the
        // chunk; SW128 stores chunk j at j ^ g.  Rows are 128 bytes, so the bank of a store depends on that chunk
        // only, and one STS.64 of 16 lanes (g = 0..3 or 4..7, t = 0..3) needs 8 distinct chunks to be a single
        // wavefront.  Storing every thread's chunk c = k at iteration k gives chunks {2 (k % 4), 2 (k % 4) + 1} ^ g:
        // rows g and g ^ 1 meet, 2 wavefronts per half-warp.  A lane with odd g therefore stores c = k ^ 2 instead:
        // its chunk is 2 (k % 4) ^ x with x = 4 (g % 2) ^ g ^ t / 2, and x takes all 8 values over the 16 lanes of
        // either half-warp (g = 0..3: {0,1} {5,4} {2,3} {7,6}; g = 4..7: {4,5} {1,0} {6,7} {3,2}), so every STS.64
        // is 2 wavefronts, one per half-warp.  c = k ^ 2 (g % 2) runs over 0..7 once, so each of the 64 x 32 float2
        // slots is written once.  The value is a register select between dq of chunks k and k ^ 2 (no dynamic
        // register index).
        const bool odd = g & 1;
        const int x = (odd ? 4 : 0) ^ g ^ (t >> 1);
        uint8_t* row = sDQ + (16 * w + g) * 128 + 8 * (t & 1);
#pragma unroll
        for (int k = 0; k < 8; ++k)
#pragma unroll
          for (int r = 0; r < 2; ++r) {
            const int e = 4 * k + 2 * r, e2 = 4 * (k ^ 2) + 2 * r;
            const float v0 = odd ? dq[e2] : dq[e], v1 = odd ? dq[e2 + 1] : dq[e + 1];
            *reinterpret_cast<float2*>(row + (k >> 2) * kDQBox + r * 8 * 128 + ((2 * (k & 3) ^ x) << 4)) =
                make_float2(v0 * p.scale, v1 * p.scale);
          }
        fence_proxy_async_smem();
        named_bar_sync(bar_id, 128);
        if (tid == 0) {
          // deterministic mode: the fp32 adds into dq_acc[query head, q block] happen in key-block order.  Key
          // block x visits Q block i iff i_begin(x) <= i < i_end(x) (neither depends on the query head); both
          // bounds grow with x, so the key blocks that visit Q block i are one run x_min..x_max, and x_min is the
          // least x with i_end(x) > i.  Without a band's lower edge x_min = 0; with one, i_end(x) > i iff 128 x +
          // 127 >= 64 i + lo, i.e. x_min = max(0, q0 + lo) / 128 (the last key block is cut at Sk, but if it is x_min
          // and misses i, no key block sees i and nobody waits).  Documents: i_end(x) is also capped by the rows of
          // the document D of x's last key c, and that cap exceeds i iff D ends after row q0, i.e. iff D is at or
          // after the document of row q0, i.e. iff c >= k_lo, the first key of row q0's document (doc_interval
          // gives it, clamped to [0, Sk], from the same boundaries): the document x_min is k_lo / 128, and x_min
          // is the larger of the two (i_end is the smaller of the two caps).  The same Sk argument holds.  Both
          // bounds still grow with x (documents never decrease along the keys), so the run stays one run.
          // The counter starts at 0, so the turn of key block x is (x - x_min) n_red + wg: x_min's first
          // reducer never waits, and each later one waits for x - 1, which visits i too.  Lower key blocks are
          // tickets of CTAs of the same (batch, K/V head) that started earlier (see the top of the kernel).  A CTA
          // visits its (query head, Q block) pairs once each, head-major and in increasing Q block order like every
          // other CTA, and only ever waits for a lower ticket; by induction over tickets (a CTA waits only for a
          // lower ticket, which by hypothesis completes all its reductions) every wait ends, so waiting for our
          // turn cannot deadlock.  The wait issues no wgmma; dK and the next S^T run on under it.
          int* turn = p.sem ? p.sem + ((int64_t)b * p.H + h) * nQ + (i_begin + it) : nullptr;
          int x_min = 0;
          if constexpr (kBand) x_min = max(0, q0 + p.lo) / kBwdN;
          if constexpr (kDoc) {
            int k_lo, unused;
            doc_interval(p.q_pos0 + p.pstride * q0, p.cu, p.n_docs, p.k_pos0, p.pstride, p.Sk, &k_lo,
                         &unused);
            x_min = max(x_min, k_lo / kBwdN);
          }
          const int my_turn = (kb - x_min) * n_red + wg;
          if (turn) {
            while (ld_acquire_gpu(turn) != my_turn) __nanosleep(64);
          }
          tma_reduce_add_4d(&tmDQ, sDQ, wg * 64, h, q0, b);
          tma_reduce_add_4d(&tmDQ, sDQ + kDQBox, wg * 64 + 32, h, q0, b);
          tma_store_commit();  // one bulk group: the wait below covers both boxes
          if (turn) {
            tma_store_wait<0>();  // our reduction has been performed ...
            __threadfence();
            st_release_gpu(turn, my_turn + 1);  // ... next turn
          }
        }
      }

      if constexpr (kNext) {
        fence_regs<32>(dp);
        issue_xt(dp, sV, do_stage(st_next));
      } else {
        wgmma_wait<0>();  // dK done
        fence_regs<kAcc>(dk);
        __syncwarp();
        if (lane == 0) mbar_arrive(&bars->q_empty[st]);
      }
      if (++it == n_it) it = 0, ++h;
      st = st_next, ph = ph_next;
    };

    for (int step = 0; step < n_steps - 1; ++step) step_body(std::true_type(), step);
    step_body(std::false_type(), n_steps - 1);
    if (kRed && tid == 0) tma_store_wait<0>();
  };
  if constexpr (kD == 128) consume(std::true_type());
  else if (wg == 0) consume(std::true_type());
  else consume(std::false_type());

  // ---------------------------------------------------------- epilogue: dk_acc += scale*dK, dv_acc += dV
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    if (keys[r] >= p.Sk) continue;
    float* pk = p.dk_acc + (int64_t)b * p.dk_sb + (int64_t)keys[r] * p.dk_ss + (int64_t)hk * p.dk_sh + 2 * t;
    float* pv = p.dv_acc + (int64_t)b * p.dv_sb + (int64_t)keys[r] * p.dv_ss + (int64_t)hk * p.dv_sh + 2 * t;
#pragma unroll
    for (int c = 0; c < kD / 8; ++c) {
      float2 a = *reinterpret_cast<float2*>(pk + 8 * c);
      a.x = fmaf(dk[4 * c + 2 * r], p.scale, a.x);
      a.y = fmaf(dk[4 * c + 2 * r + 1], p.scale, a.y);
      *reinterpret_cast<float2*>(pk + 8 * c) = a;
      float2 v = *reinterpret_cast<float2*>(pv + 8 * c);
      v.x += dv[4 * c + 2 * r];
      v.y += dv[4 * c + 2 * r + 1];
      *reinterpret_cast<float2*>(pv + 8 * c) = v;
    }
  }
}

template <bool kBF16, int kD, bool kBand>
__global__ void __launch_bounds__(kBwdThreads, 1)
bwd_chunk_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                 const __grid_constant__ CUtensorMap tmV, const __grid_constant__ CUtensorMap tmDO,
                 const __grid_constant__ CUtensorMap tmDQ, const BwdParams p) {
  bwd_chunk_body<kBF16, kD, kBand, false>(tmQ, tmK, tmV, tmDO, tmDQ, p);
}

// ALiBi instantiations: bwd_alibi_sm90.cu
template <bool kBF16, int kD, bool kBand>
__global__ void __launch_bounds__(kBwdThreads, 1)
bwd_alibi_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                 const __grid_constant__ CUtensorMap tmV, const __grid_constant__ CUtensorMap tmDO,
                 const __grid_constant__ CUtensorMap tmDQ, const BwdParams p) {
  bwd_chunk_body<kBF16, kD, kBand, true>(tmQ, tmK, tmV, tmDO, tmDQ, p);
}

// document instantiations: bwd_doc_sm90.cu
template <bool kBF16, int kD>
__global__ void __launch_bounds__(kBwdThreads, 1)
bwd_doc_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
               const __grid_constant__ CUtensorMap tmV, const __grid_constant__ CUtensorMap tmDO,
               const __grid_constant__ CUtensorMap tmDQ, const BwdParams p) {
  bwd_chunk_body<kBF16, kD, true, false, true>(tmQ, tmK, tmV, tmDO, tmDQ, p);
}

// Each tile TU instantiates its own kernels and hands bwd_chunk_run (bwd_sm90.cu), which launches every one of them,
// the kernel of a call's (dtype, head dim, ...) with the dynamic shared memory it needs.
struct BwdKernel {
  void (*fn)(CUtensorMap, CUtensorMap, CUtensorMap, CUtensorMap, CUtensorMap, BwdParams);
  int smem;
};

// bwd_chunk_kernel of (dtype, head dim) for this TU's kBand: bwd_sm90.cu kBand = false, bwd_band_sm90.cu true
template <bool kBand>
inline BwdKernel bwd_chunk_kernel_of(bool bf16, int D) {
  if (D == 64)
    return {bf16 ? bwd_chunk_kernel<true, 64, kBand> : bwd_chunk_kernel<false, 64, kBand>, BwdLayout<64>::kSmemBytes};
  return {bf16 ? bwd_chunk_kernel<true, 128, kBand> : bwd_chunk_kernel<false, 128, kBand>, BwdLayout<128>::kSmemBytes};
}

BwdKernel bwd_band_kernel_of(bool bf16, int D);              // bwd_band_sm90.cu
BwdKernel bwd_alibi_kernel_of(bool bf16, int D, bool band);  // bwd_alibi_sm90.cu
BwdKernel bwd_doc_kernel_of(bool bf16, int D);               // bwd_doc_sm90.cu

}  // namespace ba
