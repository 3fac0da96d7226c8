// seg_sync.cuh — SyncBN statistics exchange folded INTO the kernels that produce the statistics.
//
// A stand-alone exchange kernel per BatchNorm layer and direction (226 launches per DeepLab-R101 step) would be a world-wide
// flag barrier sitting alone between a conv epilogue and bn_apply, paid once per exchange.  Here the exchange has no launch
// of its own.  A producer is a kernel that ends with per-channel totals: the conv epilogues / the depthwise conv / bn_stats
// (fp64 atomics into the layer's accumulators), bn_bwd_reduce and the cooperative BN backward.  ONE block of it — the last to
// finish (one ticket per launch), or block 0 after a grid barrier — runs the whole exchange with its cooperating threads:
//   push     store the finished totals into slot[rank] of EVERY peer's symmetric buffer (P2P stores through NVSwitch);
//   publish  raise this rank's flag on every peer (st.release.sys);
//   wait     poll the world's flags in the LOCAL buffer (ld.acquire.sys);
//   total    add the world's vectors in rank order (-> bit-identical totals on every rank, no broadcast), in place;
//   advance  store the sequence number.
// The producer's ordinary output then holds the WORLD's totals, so the consumers (bn_apply, bn_bwd_apply) are the single-GPU
// kernels.  seg_comm.cu's stand-alone exchange (seg_syncbn_exchange, for callers outside the engine) is one block running
// sync_exchange_block_f.
//
// Protocol state, per rank a symmetric buffer
//     float data[2][world][n_max] | uint32 flags[2][world] | uint32 seq
// `seq` = number of exchanges this rank has COMPLETED, kept on the device (all ranks issue the same exchanges in the same
// order) so a captured CUDA graph replays correctly; epoch = seq + 1 is the flag value and its parity picks the slot.  A rank
// can run at most one exchange ahead of the slowest peer (it waits for every peer's flag of the current epoch, and a peer
// raises it only after it has read the totals of the previous epoch), so a slot is never overwritten while read.
#pragma once
#include <stdint.h>
#include <stdio.h>
#include "seg_common.cuh"

namespace seg {

// the kernels take the C handle by value; timeout_clocks <= 0 bounds the spin wait at 2^62 clocks
using SyncDesc = seg_sync_desc;

__host__ __device__ inline size_t sync_flags_offset(int world, int n_max) {
  size_t b = (size_t)2 * world * n_max * sizeof(float);
  return (b + 127) & ~(size_t)127;
}
__host__ __device__ inline size_t sync_seq_offset(int world, int n_max) {
  size_t b = sync_flags_offset(world, n_max) + (size_t)2 * world * sizeof(uint32_t);
  return (b + 127) & ~(size_t)127;
}

// Host check of the descriptor every entry point that runs the exchange makes before it launches anything (the kernels
// copy it by value and trust it).  The handle is read on the host: a device address (such as the peer-pointer array
// itself) is refused, not dereferenced.  n_max must be even: the fp64 forward statistics address slot
// (parity * world + p) * n_max FLOATS as doubles, so an odd n_max misaligns every other rank's slot and the second parity.
// `need`: floats of one rank's vector in its slot (4C for the fp64 statistics, 2C for the fp32 backward sums).
inline int sync_check_desc(const seg_sync_desc* s, int64_t need, const char* who) {
  cudaPointerAttributes attr;
  const bool host_handle = s != nullptr && cudaPointerGetAttributes(&attr, s) == cudaSuccess && attr.type != cudaMemoryTypeDevice;
  if (!host_handle) cudaGetLastError();  // a failed query must not surface at the next launch check
  SEG_REQUIRE(host_handle, "%s: `sync` must point to a seg_sync_desc in host memory", who);
  SEG_REQUIRE(s->peers != nullptr, "%s: SyncBN descriptor: peers is NULL", who);
  SEG_REQUIRE(s->world >= 1 && s->world <= 64, "%s: SyncBN descriptor: world = %d outside [1, 64]", who, s->world);
  SEG_REQUIRE(s->rank >= 0 && s->rank < s->world, "%s: SyncBN descriptor: rank = %d outside [0, world = %d)", who, s->rank,
              s->world);
  SEG_REQUIRE(s->n_max > 0 && s->n_max % 2 == 0, "%s: SyncBN descriptor: n_max = %d must be positive and even", who, s->n_max);
  SEG_REQUIRE(need > 0 && need <= s->n_max, "%s: SyncBN descriptor: n_max = %d floats cannot hold the %lld of this exchange",
              who, s->n_max, (long long)need);
  return 0;
}

__device__ __forceinline__ void sync_st_release_sys(uint32_t* p, uint32_t v) {
  asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ uint32_t sync_ld_acquire_sys(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ uint32_t sync_ld_relaxed_sys(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.relaxed.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}

// epoch of the exchange in flight on this stream (seq is advanced at the end of the previous one)
__device__ __forceinline__ uint32_t sync_epoch(const SyncDesc& s) {
  const uint32_t* seq = reinterpret_cast<const uint32_t*>(reinterpret_cast<const char*>(s.peers[s.rank]) + sync_seq_offset(s.world, s.n_max));
  uint32_t e = sync_ld_relaxed_sys(seq) + 1u;
  if (e == 0u) e = 2u;  // flags start at 0: skip it on wrap-around, keeping the parity alternation
  return e;
}

// push, per value: store element `idx` of this rank's vector into slot[rank] of every peer (myself included)
__device__ __forceinline__ void sync_push_value(const SyncDesc& s, uint32_t epoch, int idx, float v) {
  const size_t off = ((size_t)(epoch & 1u) * s.world + s.rank) * s.n_max + idx;
  for (int p = 0; p < s.world; ++p) reinterpret_cast<float*>(s.peers[p])[off] = v;
}

// the forward statistics travel as fp64 (the slot is addressed as doubles: 2 * n values need 4 * n <= n_max floats), so the
// world total is the exact sum of the ranks' exact totals and a one-rank "world" reproduces the local result bit for bit
__device__ __forceinline__ void sync_push_value_d(const SyncDesc& s, uint32_t epoch, int idx, double v) {
  const size_t off = ((size_t)(epoch & 1u) * s.world + s.rank) * s.n_max;
  for (int p = 0; p < s.world; ++p) reinterpret_cast<double*>(reinterpret_cast<float*>(s.peers[p]) + off)[idx] = v;
}
__device__ __forceinline__ double sync_total_d(const SyncDesc& s, uint32_t epoch, int idx) {
  const float* my = reinterpret_cast<const float*>(s.peers[s.rank]) + (size_t)(epoch & 1u) * s.world * s.n_max;
  double t = 0.0;
  for (int p = 0; p < s.world; ++p) t += __ldcv(reinterpret_cast<const double*>(my + (size_t)p * s.n_max) + idx);
  return t;
}

// publish, by the `nthr` cooperating threads of the exchanging block after their pushes: raise this rank's flag on every peer
template <class Sync>
__device__ __forceinline__ void sync_publish(const SyncDesc& s, uint32_t epoch, int tid, Sync sync) {
  __threadfence_system();
  sync();
  if (tid < s.world) {
    uint32_t* f = reinterpret_cast<uint32_t*>(reinterpret_cast<char*>(s.peers[tid]) + sync_flags_offset(s.world, s.n_max)) +
                  (size_t)(epoch & 1u) * s.world + s.rank;
    sync_st_release_sys(f, epoch);
  }
}

// total: world total of element idx, added in rank order (bit-identical on every rank)
__device__ __forceinline__ float sync_total(const SyncDesc& s, uint32_t epoch, int idx) {
  const float* my = reinterpret_cast<const float*>(s.peers[s.rank]) + (size_t)(epoch & 1u) * s.world * s.n_max + idx;
  float t = 0.f;
  for (int p = 0; p < s.world; ++p) t += __ldcv(my + (size_t)p * s.n_max);
  return t;
}

// wait for the world's flags with the `nthr` cooperating threads of ONE block (tid 0..nthr-1, `sync()` their barrier)
template <bool kPrint = true, class Sync>
__device__ __forceinline__ void sync_wait_world_block(const SyncDesc& s, uint32_t epoch, int tid, Sync sync) {
  if (tid < s.world) {
    const uint32_t* mine = reinterpret_cast<const uint32_t*>(reinterpret_cast<const char*>(s.peers[s.rank]) + sync_flags_offset(s.world, s.n_max)) +
                           (size_t)(epoch & 1u) * s.world + tid;
    const long long limit = s.timeout_clocks > 0 ? s.timeout_clocks : (1ll << 62);
    const long long t0 = clock64();
    while (sync_ld_acquire_sys(mine) != epoch) {
      if (clock64() - t0 > limit) {
        if constexpr (kPrint)
          printf("seg_b200: SyncBN exchange timeout (rank %d waiting for rank %d, epoch %u; raise SEG_SYNC_TIMEOUT_S)\n", s.rank, tid, epoch);
        __trap();
      }
    }
  }
  sync();
}
__device__ __forceinline__ void sync_advance(const SyncDesc& s, uint32_t epoch) {
  uint32_t* seq = reinterpret_cast<uint32_t*>(reinterpret_cast<char*>(s.peers[s.rank]) + sync_seq_offset(s.world, s.n_max));
  *seq = epoch;
  __threadfence();
}
// fp64 totals acc[0..n) (this rank's, final) -> world totals, in place; called by the cooperating threads of ONE block
template <bool kPrint, class Sync>
__device__ __forceinline__ void sync_exchange_block_d(const SyncDesc& s, double* acc, int n, int tid, int nthr, Sync sync) {
  const uint32_t epoch = sync_epoch(s);
  for (int i = tid; i < n; i += nthr) sync_push_value_d(s, epoch, i, __ldcg(acc + i));
  sync_publish(s, epoch, tid, sync);
  sync_wait_world_block<kPrint>(s, epoch, tid, sync);
  for (int i = tid; i < n; i += nthr) acc[i] = sync_total_d(s, epoch, i);
  __threadfence();
  sync();
  if (tid == 0) sync_advance(s, epoch);
}
// fp32 variant (BatchNorm backward sums, seg_syncbn_exchange)
template <class Sync>
__device__ __forceinline__ void sync_exchange_block_f(const SyncDesc& s, float* vals, int n, int tid, int nthr, Sync sync) {
  const uint32_t epoch = sync_epoch(s);
  for (int i = tid; i < n; i += nthr) sync_push_value(s, epoch, i, __ldcg(vals + i));
  sync_publish(s, epoch, tid, sync);
  sync_wait_world_block(s, epoch, tid, sync);
  for (int i = tid; i < n; i += nthr) vals[i] = sync_total(s, epoch, i);
  __threadfence();
  sync();
  if (tid == 0) sync_advance(s, epoch);
}

// producer epilogue for kernels that accumulate their per-channel totals with fp64 atomics into `acc` (n doubles): every
// contributing block calls this with its `nthr` cooperating threads after issuing its atomics; the LAST of `nblocks` blocks to
// arrive (ticket) turns the finished totals into the world's (sync_exchange_block_d).
// kPrint = false: time out with a bare trap — no printf call, which would make ptxas serialise a caller's wgmma pipeline
template <bool kPrint = true, class Sync>
__device__ __forceinline__ void sync_push_when_last(const SyncDesc& s, double* acc, int n, unsigned* ticket, unsigned nblocks,
                                                    int tid, int nthr, Sync sync, volatile int* sm_flag) {
  __threadfence();
  sync();
  if (tid == 0) *sm_flag = (atomicAdd(ticket, 1u) == nblocks - 1u);
  sync();
  if (!*sm_flag) return;
  __threadfence();
  sync_exchange_block_d<kPrint>(s, acc, n, tid, nthr, sync);
}

}  // namespace seg
