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
// Warpgroup 0 is the TMA producer (K, V once; Q, dO and the row statistics per step, 2 stages); warpgroups 1 and 2
// own 64 keys each and keep their dK, dV accumulators in registers across all G heads, so the epilogue does a
// single read-modify-write of dk_acc / dv_acc per CTA (no atomics; dK / dV stay deterministic):
//   S^T  = K_w Q_i^T,  dP^T = V_w dO_i^T      (wgmma SS m64n64, K-major operands)
//   P^T  = exp2(S^T c [+ bias] - lse2),  dS^T = P^T o (dP^T - delta)     (registers, thread = 2 key rows)
//   dV_w += P^T dO_i,  dK_w += dS^T Q_i       (wgmma RS: P^T / dS^T re-packed to 16 bit as the A operand,
//                                               dO / Q read MN-major)
//   dS^T -> smem (double-buffered), then dQ_i = dS K  (wgmma SS, both operands MN-major; head dim 128: each
//   warpgroup computes 64 of the dQ columns, head dim 64: warpgroup 1 alone) -> smem -> cp.reduce.async.bulk.tensor
//   (fp32 add in L2) into dq_acc.
// Per step a consumer warpgroup keeps its own MMAs running under its element-wise work (five commit groups; four,
// without dQ, for the non-reducing warpgroup at head dim 64):
//   issue S^T | issue dP^T | wait<1>: P^T (exp2, bias, masks) + pack, under dP^T | wait<0> | issue dV |
//   dS^T + pack + store to smem, under dV | barrier with the other warpgroup | issue dQ | issue dK |
//   wait<1> (dV, dQ done): stage dQ + reduce-add, under dK | wait<0> | release the Q / dO stage.
// The packed A operands (P^T for dV, dS^T for dK) stay untouched until the wait that retires their group.
// smem (D = 128): K 32K, V 32K, Q 2x16K, dO 2x16K, dS^T 2x16K, dQ staging 16K per reducing warpgroup (single-
// buffered: its next write waits for the previous reduce to have read it), row statistics 1K.
#include <math.h>
#include <stdlib.h>

#include <mutex>
#include <vector>

#include "host_common.h"
#include "sm90_ptx.cuh"

namespace ba {

constexpr int kBwdThreads = 384;  // warpgroup 0: loader (warp 0); warpgroups 1, 2: MMA + element-wise
constexpr int kBwdN = 128;        // keys per CTA
constexpr int kBwdM = 64;         // query rows per block of the Q-bundle
constexpr float kBwdLog2e = 1.4426950408889634f;

template <int N>
__device__ __forceinline__ void reg_inc() {
  asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(N));
}
template <int N>
__device__ __forceinline__ void reg_dec() {
  asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(N));
}

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
};

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
  uint64_t q_full[2], q_empty[2];  // Q, dO and the row statistics of one Q block
  int key_block;                   // deterministic mode: this CTA's ticket
};

// smem carve-up (bytes from the 1 KiB-aligned base); head dim kD (64 or 128)
template <int kD>
struct BwdLayout {
  static_assert(kD == 64 || kD == 128, "head dim 64 or 128");
  static constexpr int kBoxes = kD / 64;
  static constexpr int kBoxKV = kBwdN * 128;  // 16 KiB: [128 keys][64 cols] SW128 box
  static constexpr int kBoxQ = kBwdM * 128;   // 8 KiB: [64 rows][64 cols] SW128 box
  static constexpr int kOffK = 0;
  static constexpr int kOffV = kOffK + kBoxes * kBoxKV;
  static constexpr int kOffQ = kOffV + kBoxes * kBoxKV;     // 2 stages
  static constexpr int kOffDO = kOffQ + 2 * kBoxes * kBoxQ;  // 2 stages
  static constexpr int kOffDS = kOffDO + 2 * kBoxes * kBoxQ; // 2 x [128 keys][64 q] SW128
  static constexpr int kOffDQ = kOffDS + 2 * kBwdN * 128;    // per reducing warpgroup [64 rows][64] fp32
  static constexpr int kOffStat = kOffDQ + kBoxes * kBwdM * 64 * 4;  // 2 stages x [lse2 | delta] x 64 fp32
  static constexpr int kOffBar = kOffStat + 2 * 2 * kBwdM * 4;
  static constexpr int kSmemBytes = kOffBar + 64;  // no align slack: the dynamic smem base is checked to be 1 KiB aligned
  static_assert(kSmemBytes <= 232448, "backward kernel exceeds 227 KiB of shared memory");
};

template <bool kBF16, int kD>
__global__ void __launch_bounds__(kBwdThreads, 1)
bwd_chunk_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                 const __grid_constant__ CUtensorMap tmV, const __grid_constant__ CUtensorMap tmDO,
                 const __grid_constant__ CUtensorMap tmDQ, const BwdParams p) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = smem_raw;
  if ((smem_u32(smem) & 1023u) != 0) __trap();  // SWIZZLE_128B atoms need a 1 KiB-aligned base
  using L = BwdLayout<kD>;
  constexpr int kBoxes = L::kBoxes, kBoxKV = L::kBoxKV, kBoxQ = L::kBoxQ, kAcc = kD / 2;
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
  const int i_begin = p.causal ? max(0, k0 - p.causal_off) / kBwdM : 0;
  const int n_it = max(0, nQ - i_begin);
  if (n_it == 0) return;  // nothing visible: dK/dV contributions are zero (uniform exit, no barriers yet)
  const int n_steps = p.G * n_it;  // step j: query head h0 + j / n_it, Q block i_begin + j % n_it

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmQ);
    tma_prefetch_desc(&tmK);
    tma_prefetch_desc(&tmV);
    tma_prefetch_desc(&tmDO);
    tma_prefetch_desc(&tmDQ);
    mbar_init(&bars->kv_full, 1);
    for (int s = 0; s < 2; ++s) {
      mbar_init(&bars->q_full[s], 1);
      mbar_init(&bars->q_empty[s], 8);  // one elected arrive per consumer warp
    }
    fence_mbar_init();
  }
  __syncthreads();

  if (warp < 4) {
    // ============================================================ loader (warp 0)
    reg_dec<24>();
    if (warp != 0) return;
    if (lane == 0) {
      mbar_arrive_expect_tx(&bars->kv_full, 2 * kBoxes * kBoxKV);
      for (int half = 0; half < kBoxes; ++half) {
        tma_load_4d(smem + L::kOffK + half * kBoxKV, &tmK, &bars->kv_full, half * 64, hk, k0, b);
        tma_load_4d(smem + L::kOffV + half * kBoxKV, &tmV, &bars->kv_full, half * 64, hk, k0, b);
      }
    }
    int it = 0, h = h0;  // Q block (relative to i_begin) and query head of this step
    for (int step = 0; step < n_steps; ++step) {
      const int q0 = (i_begin + it) * kBwdM;
      const int st = step & 1;
      mbar_wait(&bars->q_empty[st], ((step >> 1) & 1) ^ 1);
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
        stat[lane + 32 * j] = l * kBwdLog2e;
        stat[kBwdM + lane + 32 * j] = dl;
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
    }
    return;
  }

  // ============================================================ consumers (64 keys per warpgroup)
  reg_inc<240>();
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
  const bool reducer = kD == 128 || wg == 0;  // owns 64 columns of dQ
  const int n_red = kD == 128 ? 2 : 1;

  float dk[kAcc], dv[kAcc];
#pragma unroll
  for (int i = 0; i < kAcc; ++i) dk[i] = dv[i] = 0.f;

  const uint32_t sK = smem_u32(smem + L::kOffK), sV = smem_u32(smem + L::kOffV);
  const uint32_t kw = wg * 64 * 128;  // this group's 64 key rows inside every K / V box
  float* sDQ = reinterpret_cast<float*>(smem + L::kOffDQ) + wg * kBwdM * 64;
  mbar_wait(&bars->kv_full, 0);
  int it = 0, h = h0;  // Q block (relative to i_begin) and query head of this step
  for (int step = 0; step < n_steps; ++step) {
    const int q0 = (i_begin + it) * kBwdM;
    const int st = step & 1;
    const uint32_t sQ = smem_u32(smem + L::kOffQ + st * kQStageB), sDO = smem_u32(smem + L::kOffDO + st * kQStageB);
    const float* stat = sStat + st * 2 * kBwdM;
    if (it == 0) {
#pragma unroll
      for (int r = 0; r < 2; ++r)
        bias2[r] = (p.bias && keys[r] < p.Sk)
                       ? __ldg(p.bias + (int64_t)b * p.bias_sb + (int64_t)h * p.bias_sh + keys[r]) * kBwdLog2e
                       : 0.f;
    }
    mbar_wait(&bars->q_full[st], (step >> 1) & 1);

    // S^T and dP^T as two commit groups: P^T is computed from S^T while dP^T is still running
    float s[32], dp[32];
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < kD / 16; ++kk) {
      const uint32_t okv = (kk >> 2) * kBoxKV + kw + (kk & 3) * 32, oq = (kk >> 2) * kBoxQ + (kk & 3) * 32;
      wgmma_ss_n64<kBF16, 0, 0>(s, make_desc(sK + okv, 16, 1024), make_desc(sQ + oq, 16, 1024), kk > 0 ? 1u : 0u);
    }
    wgmma_commit();
#pragma unroll
    for (int kk = 0; kk < kD / 16; ++kk) {
      const uint32_t okv = (kk >> 2) * kBoxKV + kw + (kk & 3) * 32, oq = (kk >> 2) * kBoxQ + (kk & 3) * 32;
      wgmma_ss_n64<kBF16, 0, 0>(dp, make_desc(sV + okv, 16, 1024), make_desc(sDO + oq, 16, 1024), kk > 0 ? 1u : 0u);
    }
    wgmma_commit();
    wgmma_wait<1>();  // S^T done, dP^T may still run
    fence_regs<32>(s);

    // P^T in place of S^T (fp32, kept for dS^T) and packed to 16 bit as the A operand of dV.
    // visible iff key <= q + off  <=>  q >= key - off ; whole block visible when q0 + off >= k0 + 127
    const bool need_mask = p.causal && (q0 + p.causal_off < k0 + kBwdN - 1);
    uint32_t pp[16], ds[16];
#pragma unroll
    for (int c = 0; c < 8; ++c) {
      const float2 l2 = *reinterpret_cast<const float2*>(stat + 8 * c + 2 * t);
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        const int e = 4 * c + 2 * r;
        float p0 = ex2(fmaf(s[e], scale_log2, bias2[r] - l2.x));
        float p1 = ex2(fmaf(s[e + 1], scale_log2, bias2[r] - l2.y));
        if (keys[r] >= p.Sk) p0 = p1 = 0.f;
        if (need_mask) {
          const int q = q0 + 8 * c + 2 * t;
          if (q < keys[r] - p.causal_off) p0 = 0.f;
          if (q + 1 < keys[r] - p.causal_off) p1 = 0.f;
        }
        s[e] = p0, s[e + 1] = p1;
        pp[2 * c + r] = pack2<kBF16>(p0, p1);
      }
    }

    // dV += P^T dO   (B operand: [q rows][d] tile read MN-major); pp is read by the MMA until the wait<1> below
    wgmma_wait<0>();  // dP^T done
    fence_regs<32>(dp);
    fence_regs<16>(pp);
    fence_regs<kAcc>(dv);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < kBwdM / 16; ++kk) {
      const uint64_t d_do = make_desc(sDO + kk * 16 * 128, kBoxQ, 1024);
      if constexpr (kD == 128) wgmma_rs_n128<kBF16, 1>(dv, pp + 4 * kk, d_do, 1u);
      else wgmma_rs_n64<kBF16, 1>(dv, pp + 4 * kk, d_do, 1u);
    }
    wgmma_commit();

    // dS^T = P^T o (dP^T - delta) while dV runs
#pragma unroll
    for (int c = 0; c < 8; ++c) {
      const float2 dl = *reinterpret_cast<const float2*>(stat + kBwdM + 8 * c + 2 * t);
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        const int e = 4 * c + 2 * r;
        ds[2 * c + r] = pack2<kBF16>(s[e] * (dp[e] - dl.x), s[e + 1] * (dp[e + 1] - dl.y));
      }
    }

    // dS^T -> smem [128 keys][64 q] (SW128: 16-byte chunk j of row r at j ^ (r % 8)), double-buffered: the buffer
    // written here was last read by the dQ MMAs of step - 2.  Each reducing warpgroup's wgmma_wait<1> of step - 2
    // completes its dQ group (dV and dQ are the two oldest of its three groups), and that wait comes before the
    // warpgroup reaches the barrier of step - 1, which this warpgroup has passed.
    uint8_t* sDS = smem + L::kOffDS + st * kBwdN * 128;
#pragma unroll
    for (int c = 0; c < 8; ++c)
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        const int kr = kr_lo + 8 * r;
        *reinterpret_cast<uint32_t*>(sDS + kr * 128 + ((c ^ (kr & 7)) << 4) + 4 * t) = ds[2 * c + r];
      }
    fence_proxy_async_smem();
    named_bar_sync(1, 256);

    // dQ[:, 64 wg .. 64 wg + 63] = dS K  (A = dS^T tile read MN-major, B = K tile read MN-major), then
    // dK += dS^T Q (B operand read MN-major) as the last group: it runs on under the dQ staging below
    // (head dim 64: the non-reducing warpgroup issues dK alone; each role runs its whole issue-to-wait sequence in
    // one branch, so that no wgmma group crosses a divergent path, which would make ptxas serialize them)
    float dq[32];
    fence_regs<16>(ds);
    fence_regs<kAcc>(dk);
    auto issue_dk = [&]() {
#pragma unroll
      for (int kk = 0; kk < kBwdM / 16; ++kk) {
        const uint64_t d_q = make_desc(sQ + kk * 16 * 128, kBoxQ, 1024);
        if constexpr (kD == 128) wgmma_rs_n128<kBF16, 1>(dk, ds + 4 * kk, d_q, 1u);
        else wgmma_rs_n64<kBF16, 1>(dk, ds + 4 * kk, d_q, 1u);
      }
      wgmma_commit();
    };
    if (reducer) {
      const uint32_t a0 = smem_u32(sDS), b0 = sK + wg * kBoxKV;
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < kBwdN / 16; ++kk)
        wgmma_ss_n64<kBF16, 1, 1>(dq, make_desc(a0 + kk * 16 * 128, 8192, 1024),
                                  make_desc(b0 + kk * 16 * 128, kBoxKV, 1024), kk > 0 ? 1u : 0u);
      wgmma_commit();
      issue_dk();
      wgmma_wait<1>();  // dV and dQ done, dK may still run
    } else {
      wgmma_fence();
      issue_dk();
      wgmma_wait<1>();  // dV done, dK may still run
    }
    fence_regs<kAcc>(dv);
    fence_regs<16>(pp);

    if (reducer) {
      fence_regs<32>(dq);
      const uint32_t bar_id = 2 + wg;
      if (tid == 0) tma_store_wait_read<0>();  // the previous reduce has finished reading the staging tile
      named_bar_sync(bar_id, 128);
#pragma unroll
      for (int c = 0; c < 8; ++c)
#pragma unroll
        for (int r = 0; r < 2; ++r)
          *reinterpret_cast<float2*>(sDQ + (16 * w + g + 8 * r) * 64 + 8 * c + 2 * t) =
              make_float2(dq[4 * c + 2 * r] * p.scale, dq[4 * c + 2 * r + 1] * p.scale);
      fence_proxy_async_smem();
      named_bar_sync(bar_id, 128);
      if (tid == 0) {
        // deterministic mode: the fp32 adds into dq_acc[query head, q block] happen in key-block order.  Key
        // blocks that see a given Q block are 0..x_max (i_begin does not depend on the query head), and lower
        // key blocks are tickets of CTAs of the same (batch, K/V head) that started earlier (see the top of the
        // kernel).  A CTA visits every (query head, Q block) of its group once, in the same head-major order
        // as every other CTA, and only ever waits for a lower ticket; by induction over tickets (ticket 0
        // never waits) every wait ends, so waiting for our turn cannot deadlock.
        int* turn = p.sem ? p.sem + ((int64_t)b * p.H + h) * nQ + (i_begin + it) : nullptr;
        const int my_turn = kb * n_red + wg;
        if (turn) {
          while (ld_acquire_gpu(turn) != my_turn) __nanosleep(64);
        }
        tma_reduce_add_4d(&tmDQ, sDQ, wg * 64, h, q0, b);
        tma_store_commit();
        if (turn) {
          tma_store_wait<0>();  // our reduction has been performed ...
          __threadfence();
          st_release_gpu(turn, my_turn + 1);  // ... next turn
        }
      }
    }
    wgmma_wait<0>();  // dK done: ds may be rewritten, and Q of this stage is no longer read
    fence_regs<kAcc>(dk);
    fence_regs<16>(ds);
    // Q, dO and the statistics of this stage are no longer read by this warp
    __syncwarp();
    if (lane == 0) mbar_arrive(&bars->q_empty[st]);
    if (++it == n_it) it = 0, ++h;
  }
  if (reducer && tid == 0) tma_store_wait<0>();

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

template <bool kBF16, int kD>
static int launch_bwd(const CUtensorMap& tmQ, const CUtensorMap& tmK, const CUtensorMap& tmV,
                      const CUtensorMap& tmDO, const CUtensorMap& tmDQ, const BwdParams& p, cudaStream_t stream) {
  auto kern = bwd_chunk_kernel<kBF16, kD>;
  constexpr int smem = BwdLayout<kD>::kSmemBytes;
  BA_CHECK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  dim3 grid((p.Sk + kBwdN - 1) / kBwdN, p.H / p.G, p.B);  // one CTA per (key block, K/V head, batch)
  kern<<<grid, kBwdThreads, smem, stream>>>(tmQ, tmK, tmV, tmDO, tmDQ, p);
  BA_CHECK_CUDA(cudaGetLastError());
  return BA_OK;
}

template <int kD>
static int launch_bwd_dt(int dtype, const CUtensorMap& tmQ, const CUtensorMap& tmK, const CUtensorMap& tmV,
                         const CUtensorMap& tmDO, const CUtensorMap& tmDQ, const BwdParams& p, cudaStream_t stream) {
  return dtype == BA_DTYPE_BF16 ? launch_bwd<true, kD>(tmQ, tmK, tmV, tmDO, tmDQ, p, stream)
                                : launch_bwd<false, kD>(tmQ, tmK, tmV, tmDO, tmDQ, p, stream);
}

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

static bool f32_view_ok(const ba_tensor4& t) {
  return t.ptr && (reinterpret_cast<uintptr_t>(t.ptr) & 15) == 0 && t.stride_b % 4 == 0 && t.stride_s % 4 == 0 &&
         t.stride_h % 4 == 0;
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
  using namespace ba;
  BA_REQUIRE(H_kv > 0 && H % H_kv == 0, "ba_bwd_chunk: H_kv=%d must be positive and divide H=%d", H_kv, H);
  BA_REQUIRE(D == 128 || D == 64, "ba_bwd_chunk: head dim %d unsupported (64 or 128)", D);
  BA_REQUIRE(B > 0 && Sq > 0 && Sk > 0 && H > 0, "ba_bwd_chunk: empty problem B=%d Sq=%d Sk=%d H=%d", B, Sq, Sk, H);
  BA_REQUIRE(dtype == BA_DTYPE_FP16 || dtype == BA_DTYPE_BF16, "ba_bwd_chunk: bad dtype %d", dtype);
  BA_REQUIRE(mask_mode == BA_MASK_NONE || mask_mode == BA_MASK_CAUSAL, "ba_bwd_chunk: bad mask mode %d", mask_mode);
  BA_REQUIRE(scale > 0.f && isfinite(scale), "ba_bwd_chunk: softmax scale must be positive and finite");
  BA_REQUIRE(d_o.ptr && q.ptr && k.ptr && v.ptr && delta.ptr && lse.ptr, "ba_bwd_chunk: null input");
  BA_REQUIRE(f32_view_ok(dq_acc) && f32_view_ok(dk_acc) && f32_view_ok(dv_acc),
             "ba_bwd_chunk: fp32 accumulators must be non-null, 16-byte aligned, strides multiple of 4");
  BA_REQUIRE(H <= 65535 && B <= 65535, "ba_bwd_chunk: H and B must be <= 65535");

  CUtensorMap tmQ, tmK, tmV, tmDO, tmDQ;
  const CUtensorMapDataType dt = lowp_dtype(dtype);
  int rc;
  if ((rc = make_tensor_map(&tmQ, q, B, Sq, H, D, dt, 2, 64, kBwdM, true))) return rc;
  if ((rc = make_tensor_map(&tmDO, d_o, B, Sq, H, D, dt, 2, 64, kBwdM, true))) return rc;
  if ((rc = make_tensor_map(&tmK, k, B, Sk, H_kv, D, dt, 2, 64, kBwdN, true))) return rc;
  if ((rc = make_tensor_map(&tmV, v, B, Sk, H_kv, D, dt, 2, 64, kBwdN, true))) return rc;
  // dQ reductions: [64 rows][64 fp32 columns] boxes, no swizzle (one per reducing warpgroup), H query heads
  if ((rc = make_tensor_map(&tmDQ, dq_acc, B, Sq, H, D, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, 64, kBwdM, false)))
    return rc;

  BwdParams p;
  p.lse = lse.ptr, p.lse_sb = lse.stride_b, p.lse_sh = lse.stride_h;
  p.delta = delta.ptr, p.dl_sb = delta.stride_b, p.dl_sh = delta.stride_h;
  p.dk_acc = static_cast<float*>(dk_acc.ptr);
  p.dk_sb = dk_acc.stride_b, p.dk_ss = dk_acc.stride_s, p.dk_sh = dk_acc.stride_h;
  p.dv_acc = static_cast<float*>(dv_acc.ptr);
  p.dv_sb = dv_acc.stride_b, p.dv_ss = dv_acc.stride_s, p.dv_sh = dv_acc.stride_h;
  p.bias = key_bias.ptr, p.bias_sb = key_bias.stride_b, p.bias_sh = key_bias.stride_h;
  p.B = B, p.Sq = Sq, p.Sk = Sk, p.H = H;
  p.G = H / H_kv;
  p.scale = scale;
  p.scale_log2 = scale * kBwdLog2e;
  p.causal = mask_mode == BA_MASK_CAUSAL;
  p.causal_off = causal_offset;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  p.sem = p.ticket = nullptr;
  if (flags & BA_BWD_DETERMINISTIC) {
    const size_t n_turn = (size_t)B * H * ((Sq + kBwdM - 1) / kBwdM);  // per (batch, query head, Q block)
    const size_t n = n_turn + (size_t)B * H_kv;                         // tickets per (batch, K/V head)
    p.sem = bwd_sem_workspace(n, st);
    if (p.sem) p.ticket = p.sem + n_turn;
    if (!p.sem) {
      set_error("ba_bwd_chunk: could not allocate the deterministic-mode workspace (%zu ints)", n);
      return BA_ERR_CUDA;
    }
  }
  if (D == 64) return launch_bwd_dt<64>(dtype, tmQ, tmK, tmV, tmDO, tmDQ, p, st);
  return launch_bwd_dt<128>(dtype, tmQ, tmK, tmV, tmDO, tmDQ, p, st);
}
