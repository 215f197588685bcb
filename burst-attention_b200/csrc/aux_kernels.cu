// HBM-bound helpers around the tile kernels: delta = rowsum(O*dO), fp32 -> 16-bit
// cast of the gradient accumulators, and fp32 accumulate (dQ add-on-arrival).
// All are one pass over their operands with 16-byte accesses; head dim D = 64 or 128: a (row, head) pair is
// covered by D/16 (delta), D/8 (cast) or D/4 (accumulate) consecutive threads (`lpr`, a power of two).
#include "host_common.h"
#include "sm90_ptx.cuh"

namespace ba {

// delta[b,h,s] = sum_d O[b,s,h,d] * dO[b,s,h,d]     (burst_attn_interface.py:272-278)
// D/16 lanes x 16 elements cover one row; a warp handles 32 / (D/16) consecutive (row, head) pairs.
template <bool kBF16>
__global__ void __launch_bounds__(256)
delta_kernel(const uint16_t* __restrict__ o, int64_t o_sb, int64_t o_ss, int64_t o_sh,
             const uint16_t* __restrict__ d_o, int64_t do_sb, int64_t do_ss, int64_t do_sh,
             float* __restrict__ delta, int64_t dl_sb, int64_t dl_sh, int B, int S, int H, int lpr_log2) {
  const int64_t total = (int64_t)B * S * H;  // (b, s, h) rows, h fastest
  const int64_t gid = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> lpr_log2;
  const int sub = threadIdx.x & ((1 << lpr_log2) - 1);
  float acc = 0.f;
  int b = 0, s = 0, h = 0;
  const bool valid = gid < total;
  if (valid) {
    h = gid % H;
    const int64_t bs = gid / H;
    s = bs % S;
    b = bs / S;
    const uint4* po = reinterpret_cast<const uint4*>(o + b * o_sb + s * o_ss + h * o_sh + sub * 16);
    const uint4* pd = reinterpret_cast<const uint4*>(d_o + b * do_sb + s * do_ss + h * do_sh + sub * 16);
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      uint4 a = __ldg(po + i), c = __ldg(pd + i);
      const uint32_t aw[4] = {a.x, a.y, a.z, a.w}, cw[4] = {c.x, c.y, c.z, c.w};
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        float2 fa, fc;
        if constexpr (kBF16) {
          fa = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&aw[j]));
          fc = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&cw[j]));
        } else {
          fa = __half22float2(*reinterpret_cast<const __half2*>(&aw[j]));
          fc = __half22float2(*reinterpret_cast<const __half2*>(&cw[j]));
        }
        acc = fmaf(fa.x, fc.x, acc);
        acc = fmaf(fa.y, fc.y, acc);
      }
    }
  }
  acc += __shfl_xor_sync(0xffffffffu, acc, 1);
  acc += __shfl_xor_sync(0xffffffffu, acc, 2);
  if (lpr_log2 == 3) acc += __shfl_xor_sync(0xffffffffu, acc, 4);
  if (valid && sub == 0) delta[b * dl_sb + h * dl_sh + s] = acc;
}

// dst(16-bit) = src(fp32), 8 elements per thread
template <bool kBF16>
__global__ void __launch_bounds__(256)
cast_kernel(const float* __restrict__ src, int64_t s_sb, int64_t s_ss, int64_t s_sh, uint16_t* __restrict__ dst,
            int64_t d_sb, int64_t d_ss, int64_t d_sh, int B, int S, int H, int lpr_log2) {
  const int64_t total = ((int64_t)B * S * H) << lpr_log2;  // D/8 threads per row
  const int64_t gid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (gid >= total) return;
  const int sub = gid & ((1 << lpr_log2) - 1);
  const int64_t r = gid >> lpr_log2;
  const int h = r % H;
  const int64_t bs = r / H;
  const int s = bs % S;
  const int b = bs / S;
  const float4* ps = reinterpret_cast<const float4*>(src + b * s_sb + s * s_ss + h * s_sh + sub * 8);
  const float4 x = __ldg(ps), y = __ldg(ps + 1);
  uint4 o;
  o.x = pack2<kBF16>(x.x, x.y);
  o.y = pack2<kBF16>(x.z, x.w);
  o.z = pack2<kBF16>(y.x, y.y);
  o.w = pack2<kBF16>(y.z, y.w);
  *reinterpret_cast<uint4*>(dst + b * d_sb + s * d_ss + h * d_sh + sub * 8) = o;
}

// dst(fp32) += src(fp32), 4 elements per thread
__global__ void __launch_bounds__(256)
accumulate_kernel(const float* __restrict__ src, int64_t s_sb, int64_t s_ss, int64_t s_sh, float* __restrict__ dst,
                  int64_t d_sb, int64_t d_ss, int64_t d_sh, int B, int S, int H, int lpr_log2) {
  const int64_t total = ((int64_t)B * S * H) << lpr_log2;  // D/4 threads per row
  const int64_t gid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (gid >= total) return;
  const int sub = gid & ((1 << lpr_log2) - 1);
  const int64_t r = gid >> lpr_log2;
  const int h = r % H;
  const int64_t bs = r / H;
  const int s = bs % S;
  const int b = bs / S;
  const float4 x = __ldg(reinterpret_cast<const float4*>(src + b * s_sb + s * s_ss + h * s_sh + sub * 4));
  float4* pd = reinterpret_cast<float4*>(dst + b * d_sb + s * d_ss + h * d_sh + sub * 4);
  float4 y = *pd;
  y.x += x.x, y.y += x.y, y.z += x.z, y.w += x.w;
  *pd = y;
}

}  // namespace ba

extern "C" int ba_bwd_delta(ba_tensor4 o, ba_tensor4 d_o, ba_rowstat delta, int B, int S, int H, int D, int dtype,
                            void* stream) {
  using namespace ba;
  BA_REQUIRE(D == 128 || D == 64, "ba_bwd_delta: head dim %d unsupported (64 or 128)", D);
  const int lpr_log2 = D == 128 ? 3 : 2;
  BA_REQUIRE(B > 0 && S > 0 && H > 0, "ba_bwd_delta: empty problem");
  BA_REQUIRE(o.ptr && d_o.ptr && delta.ptr, "ba_bwd_delta: null pointer");
  BA_REQUIRE(aligned16(o, 2) && aligned16(d_o, 2), "ba_bwd_delta: o/dO must be 16-byte aligned views");
  const int64_t rows = (int64_t)B * S * H;
  const int64_t threads = rows << lpr_log2;
  const unsigned blocks = (unsigned)((threads + 255) / 256);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (dtype == BA_DTYPE_BF16)
    delta_kernel<true><<<blocks, 256, 0, st>>>((const uint16_t*)o.ptr, o.stride_b, o.stride_s, o.stride_h,
                                               (const uint16_t*)d_o.ptr, d_o.stride_b, d_o.stride_s, d_o.stride_h,
                                               delta.ptr, delta.stride_b, delta.stride_h, B, S, H, lpr_log2);
  else
    delta_kernel<false><<<blocks, 256, 0, st>>>((const uint16_t*)o.ptr, o.stride_b, o.stride_s, o.stride_h,
                                                (const uint16_t*)d_o.ptr, d_o.stride_b, d_o.stride_s, d_o.stride_h,
                                                delta.ptr, delta.stride_b, delta.stride_h, B, S, H, lpr_log2);
  BA_CHECK_CUDA(cudaGetLastError());
  return BA_OK;
}

extern "C" int ba_cast_from_f32(ba_tensor4 src, ba_tensor4 dst, int B, int S, int H, int D, int dtype,
                                void* stream) {
  using namespace ba;
  BA_REQUIRE(D == 128 || D == 64, "ba_cast_from_f32: head dim %d unsupported (64 or 128)", D);
  const int lpr_log2 = D == 128 ? 4 : 3;
  BA_REQUIRE(B > 0 && S > 0 && H > 0 && src.ptr && dst.ptr, "ba_cast_from_f32: bad arguments");
  BA_REQUIRE(aligned16(src, 4) && aligned16(dst, 2), "ba_cast_from_f32: views must be 16-byte aligned");
  const int64_t threads = ((int64_t)B * S * H) << lpr_log2;
  const unsigned blocks = (unsigned)((threads + 255) / 256);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (dtype == BA_DTYPE_BF16)
    cast_kernel<true><<<blocks, 256, 0, st>>>((const float*)src.ptr, src.stride_b, src.stride_s, src.stride_h,
                                              (uint16_t*)dst.ptr, dst.stride_b, dst.stride_s, dst.stride_h, B, S, H, lpr_log2);
  else
    cast_kernel<false><<<blocks, 256, 0, st>>>((const float*)src.ptr, src.stride_b, src.stride_s, src.stride_h,
                                               (uint16_t*)dst.ptr, dst.stride_b, dst.stride_s, dst.stride_h, B, S, H, lpr_log2);
  BA_CHECK_CUDA(cudaGetLastError());
  return BA_OK;
}

extern "C" int ba_accumulate_f32(ba_tensor4 src, ba_tensor4 dst, int B, int S, int H, int D, void* stream) {
  using namespace ba;
  BA_REQUIRE(D == 128 || D == 64, "ba_accumulate_f32: head dim %d unsupported (64 or 128)", D);
  const int lpr_log2 = D == 128 ? 5 : 4;
  BA_REQUIRE(B > 0 && S > 0 && H > 0 && src.ptr && dst.ptr, "ba_accumulate_f32: bad arguments");
  BA_REQUIRE(aligned16(src, 4) && aligned16(dst, 4), "ba_accumulate_f32: views must be 16-byte aligned");
  const int64_t threads = ((int64_t)B * S * H) << lpr_log2;
  const unsigned blocks = (unsigned)((threads + 255) / 256);
  accumulate_kernel<<<blocks, 256, 0, static_cast<cudaStream_t>(stream)>>>(
      (const float*)src.ptr, src.stride_b, src.stride_s, src.stride_h, (float*)dst.ptr, dst.stride_b, dst.stride_s,
      dst.stride_h, B, S, H, lpr_log2);
  BA_CHECK_CUDA(cudaGetLastError());
  return BA_OK;
}
