// Thin inline-PTX layer for sm_90a: mbarrier, TMA (cp.async.bulk.tensor),
// warpgroup MMA (wgmma.mma_async) and its shared-memory matrix descriptors.
// Hand-written for this project; bit layouts follow the PTX ISA tables for
// the wgmma matrix descriptor and register fragments.
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace ba {

#define BA_DEVICE __device__ __forceinline__

// ------------------------------------------------------------------ misc
BA_DEVICE uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
constexpr float kLog2e = 1.4426950408889634f;
constexpr float kLn2 = 0.6931471805599453f;
BA_DEVICE float ex2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
BA_DEVICE float lg2(float x) {
  float y;
  asm("lg2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
// Warp-specialised kernels hand registers from the producer warpgroup to the consumers.
template <int N>
BA_DEVICE void reg_alloc_inc() {
  asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(N));
}
template <int N>
BA_DEVICE void reg_alloc_dec() {
  asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(N));
}

// ------------------------------------------------------------------ mbarrier
BA_DEVICE void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
BA_DEVICE void fence_mbar_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
BA_DEVICE void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
BA_DEVICE void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
               : "memory");
}
BA_DEVICE bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}\n"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
// Bounded wait: a protocol bug traps after ~30 s (-> CUDA error surfaced to the
// host at its next synchronize) instead of hanging the GPU.  The watchdog must
// make no function call: a call (printf -> vprintf) inside a kernel that issues
// wgmma makes ptxas serialize every wgmma of that kernel (warning C7510), which
// the build refuses.  To locate a fault, add a printf here while debugging.
BA_DEVICE uint64_t global_ns() {
  uint64_t t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}
BA_DEVICE void mbar_wait(uint64_t* bar, uint32_t parity) {
  if (mbar_try_wait(bar, parity)) return;
#ifdef BA_NO_WATCHDOG
  while (!mbar_try_wait(bar, parity)) {
  }
#else
  const uint64_t t0 = global_ns();
#pragma unroll 1
  for (;;) {
#pragma unroll 1
    for (int i = 0; i < 1024; ++i)
      if (mbar_try_wait(bar, parity)) return;
    if (global_ns() - t0 > 30000000000ull) break;
  }
  __trap();
#endif
}

// ------------------------------------------------------------------ fences
BA_DEVICE void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
BA_DEVICE void named_bar_sync(uint32_t id, uint32_t nthreads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}

// ------------------------------------------------------------------ TMA
BA_DEVICE void tma_prefetch_desc(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
// 4-D tiled load: coordinates innermost-first (d, h, s, b).
BA_DEVICE void tma_load_4d(void* smem_dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1, int c2,
                           int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4, %5, %6}], [%2];"
      :
      : "r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1),
        "r"(c2), "r"(c3)
      : "memory");
}
// 4-D tiled reduce-add smem -> global (fp32 add performed by the TMA unit / L2).
BA_DEVICE void tma_reduce_add_4d(const CUtensorMap* m, const void* smem_src, int c0, int c1, int c2, int c3) {
  asm volatile(
      "cp.reduce.async.bulk.tensor.4d.global.shared::cta.add.tile.bulk_group [%0, {%2, %3, %4, %5}], [%1];"
      :
      : "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(smem_src)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}
BA_DEVICE void tma_store_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
template <int N>
BA_DEVICE void tma_store_wait_read() {
  asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory");
}
template <int N>
BA_DEVICE void tma_store_wait() {
  asm volatile("cp.async.bulk.wait_group %0;" ::"n"(N) : "memory");
}

// ------------------------------------------------------------------ wgmma
// Shared-memory matrix descriptor (64 bit):
//  [0,14)  start address >> 4        [16,30) leading-dim byte offset (LBO) >> 4
//  [32,46) stride-dim byte offset (SBO) >> 4   [49,52) base offset (0: atoms are 1024-B aligned)
//  [62,64) layout: 1 = 128B swizzle
// Every operand tile here is a stack of TMA boxes of [rows][64 16-bit columns] in SWIZZLE_128B (a 128-B row per
// tile row, 8-row atoms of 1 KiB):
//   K-major (the 64 columns are the K dimension): SBO = 1024 (next 8 rows of M/N), LBO unused; a K = 16 step
//     inside a box advances the start address by 32 B, the next box by the box size.
//   MN-major (the 64 columns are M or N, the rows are K): SBO = 1024 (next 8 K rows), LBO = byte distance between
//     64-wide M/N blocks (the box size); a K = 16 step advances the start address by 16 rows = 2 KiB.
BA_DEVICE uint64_t make_desc(uint32_t smem_addr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((smem_addr & 0x3FFFF) >> 4);
  d |= static_cast<uint64_t>((lbo_bytes >> 4) & 0x3FFF) << 16;
  d |= static_cast<uint64_t>((sbo_bytes >> 4) & 0x3FFF) << 32;
  d |= static_cast<uint64_t>(1) << 62;  // SWIZZLE_128B
  return d;
}

BA_DEVICE void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
BA_DEVICE void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
BA_DEVICE void wgmma_wait() {
  asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}
// Keeps the compiler from moving reads / writes of accumulator registers across a wgmma fence or wait.
template <int N>
BA_DEVICE void fence_regs(float* r) {
#pragma unroll
  for (int i = 0; i < N; ++i) asm volatile("" : "+f"(r[i])::"memory");
}
template <int N>
BA_DEVICE void fence_regs(uint32_t* r) {
#pragma unroll
  for (int i = 0; i < N; ++i) asm volatile("" : "+r"(r[i])::"memory");
}

// m64nNk16 with fp32 accumulators, one warpgroup.  Accumulator fragment of thread (warp w, lane l) of the
// warpgroup, g = l / 4, t = l % 4, for each 8-column chunk c:
//   d[4c+0], d[4c+1] -> row 16w + g,     columns 8c + 2t, 8c + 2t + 1
//   d[4c+2], d[4c+3] -> row 16w + g + 8, the same columns
// A fragment of the register form (K = 16 step kk of a 16-bit matrix laid out like an accumulator):
//   a[0..3] = pack(d[8kk+0], d[8kk+1]), pack(d[8kk+2], d[8kk+3]), pack(d[8kk+4], d[8kk+5]), pack(d[8kk+6], d[8kk+7])
// kTA / kTB: 0 = K-major, 1 = MN-major operand.  scale_d = 0 overwrites the accumulator.
// The N / 2 accumulator operands d[0 ..] of m64nNk16 and their PTX register list.
#define BA_WGMMA_ACC_64(d) "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
#define BA_WGMMA_ACC_128(d) BA_WGMMA_ACC_64(d), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
#define BA_WGMMA_REGS_64 "%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31"
#define BA_WGMMA_REGS_128 BA_WGMMA_REGS_64 ",%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63"
// The two forms, for width N and PTX type TY ("bf16" / "f16").  The numbers name the operands that follow the
// accumulators: the A descriptor (SS) or the four A registers (RS), the B descriptor, scale_d, kTA (SS) and kTB.
#define BA_WGMMA_SS(N, TY, A, B, SC, TA, TB)                                                     \
  asm volatile("{\n\t.reg .pred p;\n\t"                                                        \
               "setp.ne.b32 p, %" #SC ", 0;\n\t"                                               \
               "wgmma.mma_async.sync.aligned.m64n" #N "k16.f32." TY "." TY " "                 \
               "{" BA_WGMMA_REGS_##N "}, "                                                      \
               "%" #A ", %" #B ", p, 1, 1, %" #TA ", %" #TB ";\n\t}\n"                         \
               : BA_WGMMA_ACC_##N(d)                                                            \
               : "l"(a_desc), "l"(b_desc), "r"(scale_d), "n"(kTA), "n"(kTB))
#define BA_WGMMA_RS(N, TY, A0, A1, A2, A3, B, SC, TB)                                            \
  asm volatile("{\n\t.reg .pred p;\n\t"                                                        \
               "setp.ne.b32 p, %" #SC ", 0;\n\t"                                               \
               "wgmma.mma_async.sync.aligned.m64n" #N "k16.f32." TY "." TY " "                 \
               "{" BA_WGMMA_REGS_##N "}, "                                                      \
               "{%" #A0 ",%" #A1 ",%" #A2 ",%" #A3 "}, %" #B ", p, 1, 1, %" #TB ";\n\t}\n"     \
               : BA_WGMMA_ACC_##N(d)                                                            \
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b_desc), "r"(scale_d), "n"(kTB))

template <bool kBF16, int kTA, int kTB>
BA_DEVICE void wgmma_ss_n64(float* d, uint64_t a_desc, uint64_t b_desc, uint32_t scale_d) {
  if constexpr (kBF16) BA_WGMMA_SS(64, "bf16", 32, 33, 34, 35, 36);
  else BA_WGMMA_SS(64, "f16", 32, 33, 34, 35, 36);
}
template <bool kBF16, int kTB>
BA_DEVICE void wgmma_rs_n64(float* d, const uint32_t* a, uint64_t b_desc, uint32_t scale_d) {
  if constexpr (kBF16) BA_WGMMA_RS(64, "bf16", 32, 33, 34, 35, 36, 37, 38);
  else BA_WGMMA_RS(64, "f16", 32, 33, 34, 35, 36, 37, 38);
}
template <bool kBF16, int kTA, int kTB>
BA_DEVICE void wgmma_ss_n128(float* d, uint64_t a_desc, uint64_t b_desc, uint32_t scale_d) {
  if constexpr (kBF16) BA_WGMMA_SS(128, "bf16", 64, 65, 66, 67, 68);
  else BA_WGMMA_SS(128, "f16", 64, 65, 66, 67, 68);
}
template <bool kBF16, int kTB>
BA_DEVICE void wgmma_rs_n128(float* d, const uint32_t* a, uint64_t b_desc, uint32_t scale_d) {
  if constexpr (kBF16) BA_WGMMA_RS(128, "bf16", 64, 65, 66, 67, 68, 69, 70);
  else BA_WGMMA_RS(128, "f16", 64, 65, 66, 67, 68, 69, 70);
}

// ------------------------------------------------------------------ packing
template <bool kBF16>
BA_DEVICE uint32_t pack2(float lo, float hi) {
  if constexpr (kBF16) {
    __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);
    return *reinterpret_cast<uint32_t*>(&v);
  } else {
    __half2 v = __floats2half2_rn(lo, hi);
    return *reinterpret_cast<uint32_t*>(&v);
  }
}

}  // namespace ba
