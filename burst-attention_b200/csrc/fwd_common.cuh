// Constants and parameters of the forward tile kernel (fwd_sm90.cu).
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace ba {

constexpr int kBlockM = 128;  // Q rows per CTA (64 per consumer warpgroup)
constexpr int kBlockN = 128;  // keys per K/V tile
constexpr int kKStages = 2;
constexpr int kVStages = 2;
constexpr int kBoxBytes = 128 * 64 * 2;  // 16 KiB: one 128 x 64 SW128 TMA box (a [128][head_dim] tile is head_dim/64 boxes)
constexpr int kFwdThreads = 384;         // warpgroup 0: TMA producer; warpgroups 1, 2: MMA + softmax
constexpr float kLog2e = 1.4426950408889634f;
constexpr float kLn2 = 0.6931471805599453f;

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
};


}  // namespace ba
