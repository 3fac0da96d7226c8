// seg_comm.cu — symmetric buffers of the SyncBN statistics exchange and its stand-alone form.
//
// Replaces the reference's per-layer master-reduce + broadcast (utils/sync_batchnorm/batchnorm.py:105-126:
// ReduceAddCoalesced.apply at :117, Broadcast.apply at :120, thread pipes in comm.py) — two collectives and a Python
// queue round trip per BN layer.  The protocol (push into every peer's slot, release flags, acquire wait, rank-ordered sum,
// device-side sequence number) and the buffer layout live in seg_sync.cuh; the engine's kernels run it in their last block.
// seg_syncbn_exchange is the same exchange as a one-block launch, for callers outside the engine.
//
// Symmetric buffer layout (per rank, allocated by seg_comm_alloc, exported with CUDA IPC):
//   float    data [2][world][n_max]
//   uint32_t flags[2][world]         (at byte offset 2*world*n_max*4, 128-byte aligned)
//   uint32_t seq                     (next 128-byte line; number of exchanges this rank has completed)
#include "seg_common.cuh"
#include "seg_sync.cuh"

namespace seg {

static_assert(sizeof(seg_sync_desc) == 32, "seg_sync_desc: pointer, three int32, padding, int64 (lib.SyncDesc mirrors it)");

__global__ void __launch_bounds__(1024) syncbn_exchange_kernel(const SyncDesc s, float* __restrict__ vals, int n) {
  sync_exchange_block_f(s, vals, n, (int)threadIdx.x, (int)blockDim.x, [] { __syncthreads(); });
}

}  // namespace seg

using namespace seg;

extern "C" {

size_t seg_comm_buffer_bytes(int world, int n_max) { return sync_seq_offset(world, n_max) + 128; }

int seg_comm_alloc(size_t bytes, void** ptr) {
  cudaError_t e = cudaMalloc(ptr, bytes);
  SEG_REQUIRE(e == cudaSuccess, "seg_comm_alloc: %s", cudaGetErrorString(e));
  e = cudaMemset(*ptr, 0, bytes);
  SEG_REQUIRE(e == cudaSuccess, "seg_comm_alloc memset: %s", cudaGetErrorString(e));
  return 0;
}
int seg_comm_free(void* ptr) {
  cudaError_t e = cudaFree(ptr);
  SEG_REQUIRE(e == cudaSuccess, "seg_comm_free: %s", cudaGetErrorString(e));
  return 0;
}
int seg_comm_ipc_get(void* ptr, void* handle64) {
  static_assert(sizeof(cudaIpcMemHandle_t) == 64, "ipc handle size");
  cudaError_t e = cudaIpcGetMemHandle(reinterpret_cast<cudaIpcMemHandle_t*>(handle64), ptr);
  SEG_REQUIRE(e == cudaSuccess, "cudaIpcGetMemHandle: %s", cudaGetErrorString(e));
  return 0;
}
int seg_comm_ipc_open(const void* handle64, void** ptr) {
  cudaIpcMemHandle_t h;
  memcpy(&h, handle64, 64);
  cudaError_t e = cudaIpcOpenMemHandle(ptr, h, cudaIpcMemLazyEnablePeerAccess);
  SEG_REQUIRE(e == cudaSuccess, "cudaIpcOpenMemHandle: %s", cudaGetErrorString(e));
  return 0;
}
int seg_comm_ipc_close(void* ptr) {
  cudaError_t e = cudaIpcCloseMemHandle(ptr);
  SEG_REQUIRE(e == cudaSuccess, "cudaIpcCloseMemHandle: %s", cudaGetErrorString(e));
  return 0;
}

int seg_syncbn_exchange(const seg_sync_desc* sync, float* vals, int n, void* stream) {
  if (sync_check_desc(sync, n, "syncbn exchange")) return 1;
  // >= 64 threads: thread p < world raises this rank's flag on peer p and waits for peer p's
  const int threads = n >= 1024 ? 1024 : ((n + 31) / 32 * 32 < 64 ? 64 : (n + 31) / 32 * 32);
  syncbn_exchange_kernel<<<1, threads, 0, reinterpret_cast<cudaStream_t>(stream)>>>(*sync, vals, n);
  return check_launch("syncbn_exchange");
}

}  // extern "C"
