// Copy-engine ring transport (optional, same-node rings): one hop = peer cudaMemcpyAsync pushes over
// NVLink executed by the copy engines -- no SMs, so the hop does not compete with the tile kernels the
// way NCCL's SM-resident send/recv kernels do (which matters most for short shards, where the hop is
// exposed).  Same post/wait contract as the NCCL transport (ring_nccl.cu).
//
// Receive buffers live in a ring-owned arena that every rank carves identically (a symmetric heap), so
// "my destination's offset in my arena" is also the offset to write at in the next rank's arena, which
// is mapped here with CUDA IPC.  Flow control is two monotonic hop counters per rank kept in the arena's
// first page and awaited with cuStreamWaitValue32 (no host involvement, no kernels):
//
//   side stream, hop k:   wait(compute event)                         sources ready, destinations consumed
//                         prev.ready   <- k                           "you may overwrite my slots"
//                         wait(local.ready   >= k)                    next rank said the same to me
//                         next.arena[off_i] <- src_i   (i = 0..n-1)   copy engines over NVLink
//                         next.arrived <- k                           stream order: after the data
//                         wait(local.arrived >= k)                    my own inbound data is complete
//                         record(done event)                          ba_ring_wait makes compute wait on it
//
// Every rank announces readiness before it waits for anything remote, so the chain cannot deadlock.
#include <stdlib.h>
#include <string.h>

#include <mutex>

#include "ring_internal.h"

namespace ba {

typedef CUresult (*stream_value32_fn)(CUstream, CUdeviceptr, cuuint32_t, unsigned int);
static stream_value32_fn g_wait32 = nullptr, g_write32 = nullptr;

static bool load_memops() {
  static std::once_flag once;
  std::call_once(once, [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuStreamWaitValue32", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      g_wait32 = reinterpret_cast<stream_value32_fn>(p);
    p = nullptr;
    if (cudaGetDriverEntryPoint("cuStreamWriteValue32", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      g_write32 = reinterpret_cast<stream_value32_fn>(p);
  });
  return g_wait32 != nullptr && g_write32 != nullptr;
}

static int cu_fail(CUresult r, const char* what) {
  set_error("CUDA driver error %d at %s", static_cast<int>(r), what);
  return BA_ERR_CUDA;
}
#define BA_CHECK_CU(expr)                                 \
  do {                                                    \
    CUresult _r = (expr);                                 \
    if (_r != CUDA_SUCCESS) return ::ba::cu_fail(_r, #expr); \
  } while (0)

static int remote_flag(ba_ring* r, uint8_t* remote, uint32_t k) {
  CeState& ce = r->ce;
  if (ce.write_value) {
    BA_CHECK_CU(g_write32(r->side, reinterpret_cast<CUdeviceptr>(remote), k, 0));
  } else {
    ce.host_vals[k % kCeVals] = k;
    BA_CHECK_CUDA(cudaMemcpyAsync(remote, &ce.host_vals[k % kCeVals], 4, cudaMemcpyDefault, r->side));
  }
  return BA_OK;
}

int ce_post(ba_ring* r, const void* const* src, void* const* dst, const int64_t* nbytes, int n) {
  CeState& ce = r->ce;
  uint8_t* data = ce.base + kCeHeader;
  for (int i = 0; i < n; ++i) {
    const uint8_t* d = static_cast<const uint8_t*>(dst[i]);
    BA_REQUIRE(nbytes[i] >= 0 && d >= data && d + nbytes[i] <= data + ce.bytes,
               "ba_ring_post: destination %d is not inside the ring's receive arena (copy-engine transport)", i);
  }
  const uint32_t k = ++ce.hop;
  int rc = remote_flag(r, ce.prev_map + kCeOffReady, k);
  if (rc != BA_OK) return rc;
  BA_CHECK_CU(g_wait32(r->side, reinterpret_cast<CUdeviceptr>(ce.base + kCeOffReady), k, CU_STREAM_WAIT_VALUE_GEQ));
  for (int i = 0; i < n; ++i) {
    const int64_t off = static_cast<const uint8_t*>(dst[i]) - ce.base;
    BA_CHECK_CUDA(cudaMemcpyAsync(ce.next_map + off, src[i], (size_t)nbytes[i], cudaMemcpyDefault, r->side));
  }
  rc = remote_flag(r, ce.next_map + kCeOffArrived, k);
  if (rc != BA_OK) return rc;
  BA_CHECK_CU(g_wait32(r->side, reinterpret_cast<CUdeviceptr>(ce.base + kCeOffArrived), k, CU_STREAM_WAIT_VALUE_GEQ));
  return BA_OK;
}

// Unmap the neighbours' arenas and RETIRE (not free) the local one: a neighbour may still have it mapped, and
// freeing exported memory before every importer has closed it is undefined.  The retired arena is freed in
// ba_ring_arena_connect, which the host calls only after a collective that every rank enters after its own
// ba_ring_arena_create -- i.e. after every importer has closed its mapping.
static void ce_disconnect(ba_ring* r) {
  CeState& ce = r->ce;
  if (r->side) cudaStreamSynchronize(r->side);
  if (ce.next_map) cudaIpcCloseMemHandle(ce.next_map);
  if (ce.prev_map && ce.prev_map != ce.next_map) cudaIpcCloseMemHandle(ce.prev_map);
  if (ce.retired) cudaFree(ce.retired);  // two growths ago: long unmapped everywhere
  ce.retired = ce.base;
  ce.base = ce.next_map = ce.prev_map = nullptr;
  ce.bytes = 0;
  ce.hop = 0;
  ce.connected = false;
}

void ce_destroy(ba_ring* r) {
  ce_disconnect(r);
  if (r->ce.retired) cudaFree(r->ce.retired);
  r->ce.retired = nullptr;
  if (r->ce.host_vals) cudaFreeHost(r->ce.host_vals);
  r->ce.host_vals = nullptr;
}

}  // namespace ba

extern "C" int ba_ring_arena_create(ba_ring* ring, int64_t bytes, void** base_out, void* handle_out64) {
  using namespace ba;
  BA_REQUIRE(ring && base_out && handle_out64 && bytes > 0, "ba_ring_arena_create: bad arguments");
  BA_REQUIRE(ring->world > 1, "ba_ring_arena_create: a ring of one rank has no neighbours to map");
  static_assert(sizeof(cudaIpcMemHandle_t) == BA_IPC_HANDLE_BYTES, "IPC handle size");
  if (!load_memops()) {
    set_error("cuStreamWaitValue32 / cuStreamWriteValue32 driver entry points not available");
    return BA_ERR_UNSUPPORTED;
  }
  ce_disconnect(ring);  // the caller has quiesced every rank (see burst_attn/comm.py)
  CeState& ce = ring->ce;
  bytes = (bytes + 1023) / 1024 * 1024;
  BA_CHECK_CUDA(cudaMalloc(reinterpret_cast<void**>(&ce.base), (size_t)(bytes + kCeHeader)));
  BA_CHECK_CUDA(cudaMemset(ce.base, 0, (size_t)kCeHeader));
  BA_CHECK_CUDA(cudaDeviceSynchronize());
  ce.bytes = bytes;
  if (!ce.host_vals) BA_CHECK_CUDA(cudaMallocHost(reinterpret_cast<void**>(&ce.host_vals), kCeVals * sizeof(uint32_t)));
  const char* f = getenv("BA_CE_FLAG");
  ce.write_value = f && strcmp(f, "wv") == 0;
  cudaIpcMemHandle_t h;
  BA_CHECK_CUDA(cudaIpcGetMemHandle(&h, ce.base));
  memcpy(handle_out64, &h, sizeof(h));
  *base_out = ce.base + kCeHeader;
  return BA_OK;
}

extern "C" int ba_ring_arena_connect(ba_ring* ring, const void* prev_handle64, const void* next_handle64) {
  using namespace ba;
  BA_REQUIRE(ring && prev_handle64 && next_handle64, "ba_ring_arena_connect: bad arguments");
  CeState& ce = ring->ce;
  BA_REQUIRE(ce.base && !ce.connected, "ba_ring_arena_connect: call ba_ring_arena_create first (once per arena)");
  cudaIpcMemHandle_t hp, hn;
  memcpy(&hp, prev_handle64, sizeof(hp));
  memcpy(&hn, next_handle64, sizeof(hn));
  BA_CHECK_CUDA(cudaIpcOpenMemHandle(reinterpret_cast<void**>(&ce.next_map), hn, cudaIpcMemLazyEnablePeerAccess));
  if (memcmp(&hp, &hn, sizeof(hp)) == 0) {
    ce.prev_map = ce.next_map;  // world == 2: one neighbour, one mapping
  } else {
    BA_CHECK_CUDA(cudaIpcOpenMemHandle(reinterpret_cast<void**>(&ce.prev_map), hp, cudaIpcMemLazyEnablePeerAccess));
  }
  if (ce.retired) {  // every rank has been through its ba_ring_arena_create: nobody maps the old arena any more
    BA_CHECK_CUDA(cudaFree(ce.retired));
    ce.retired = nullptr;
  }
  ce.hop = 0;
  ce.connected = true;
  return BA_OK;
}
