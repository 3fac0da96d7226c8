// seg_sync.cuh — SyncBN statistics exchange folded INTO the kernels that produce and consume the statistics.
//
// A stand-alone exchange kernel per BatchNorm layer and direction (226 launches per DeepLab-R101 step) would be a world-wide
// flag barrier sitting alone between a conv epilogue and bn_apply, paid once per exchange.  Here the exchange has no launch
// of its own:
//
//   producer  = a kernel that ends with per-channel totals: the conv epilogues / the depthwise conv / bn_stats (fp64 atomics
//               into the layer's accumulators) and bn_bwd_reduce / the cooperative BN backward.  The LAST block to finish
//               (one ticket per launch) reads the finished totals and stores them into slot[rank] of EVERY peer's symmetric
//               buffer (P2P stores through NVSwitch), then raises this rank's flag on every peer (st.release.sys).  The NVLink
//               latency overlaps the kernel's tail and the next launch.
//   consumer  = the prologue of bn_apply / bn_bwd_apply: every block waits for the world's flags (ld.acquire.sys), then each
//               thread adds, in rank order (-> bit-identical totals on every rank, no broadcast), the world's sums for its own
//               channels from the LOCAL symmetric buffer.  The last consumer block to finish advances the sequence number.
//
// Protocol state is the same as seg_comm.cu's stand-alone exchange kernel (kept for tests and callers outside the engine): per
// rank a symmetric buffer
//     float data[2][world][n_max] | uint32 flags[2][world] | uint32 seq
// `seq` = number of exchanges this rank has COMPLETED, kept on the device (all ranks issue the same exchanges in the same
// order) so a captured CUDA graph replays correctly; epoch = seq + 1 is the flag value and its parity picks the slot.  A rank
// can run at most one exchange ahead of the slowest peer (its consumer needs every peer's flag of the current epoch, and a
// peer raises it only after ITS consumer of the previous epoch has finished), so a slot is never overwritten while read.
#pragma once
#include <stdint.h>
#include <stdio.h>

namespace seg {

struct SyncDesc {  // mirror of seg_sync_desc (include/seg_b200.h)
  void* const* peers;        // device array of `world` symmetric-buffer base pointers (peers[rank] = mine)
  int rank, world, n_max;
  long long timeout_clocks;  // spin-wait bound (<= 0: 2^62)
  int mode;                  // 0: the CONSUMER kernel waits for the world and sums (every block polls the flags);
                             // 1: the PRODUCER's last block does the whole exchange and leaves the world totals in the local buffer
};

__host__ __device__ inline size_t sync_flags_offset(int world, int n_max) {
  size_t b = (size_t)2 * world * n_max * sizeof(float);
  return (b + 127) & ~(size_t)127;
}
__host__ __device__ inline size_t sync_seq_offset(int world, int n_max) {
  size_t b = sync_flags_offset(world, n_max) + (size_t)2 * world * sizeof(uint32_t);
  return (b + 127) & ~(size_t)127;
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

// epoch of the exchange in flight on this stream (seq is advanced by the last consumer block of the previous one)
__device__ __forceinline__ uint32_t sync_epoch(const SyncDesc& s) {
  const uint32_t* seq = reinterpret_cast<const uint32_t*>(reinterpret_cast<const char*>(s.peers[s.rank]) + sync_seq_offset(s.world, s.n_max));
  uint32_t e = sync_ld_relaxed_sys(seq) + 1u;
  if (e == 0u) e = 2u;  // flags start at 0: skip it on wrap-around, keeping the parity alternation
  return e;
}

// producer, per value: store element `idx` of this rank's vector into slot[rank] of every peer (myself included)
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

// producer, once per layer, by the `nthr` cooperating threads of the block that completed the layer's LAST lane (every
// pushing block executed __threadfence_system() before taking the lane ticket): raise this rank's flag on every peer
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

// producer epilogue for kernels that accumulate their per-channel totals with fp64 atomics into `acc` (n doubles): every
// contributing block calls this with its `nthr` cooperating threads after issuing its atomics; the LAST of `nblocks` blocks to
// arrive (ticket) reads the finished totals and pushes them (as fp64) to every peer, then raises the flags.
template <bool kPrint, class Sync>
__device__ __forceinline__ void sync_exchange_block_d(const SyncDesc& s, double* acc, int n, int tid, int nthr, Sync sync);
// kPrint = false: time out with a bare trap — no printf call, which would make ptxas serialise a caller's wgmma pipeline
template <bool kPrint = true, class Sync>
__device__ __forceinline__ void sync_push_when_last(const SyncDesc& s, const double* acc, int n, unsigned* ticket, unsigned nblocks,
                                                    int tid, int nthr, Sync sync, volatile int* sm_flag) {
  __threadfence();
  sync();
  if (tid == 0) *sm_flag = (atomicAdd(ticket, 1u) == nblocks - 1u);
  sync();
  if (!*sm_flag) return;
  __threadfence();
  if (s.mode == 1) {  // the whole exchange here: acc becomes the world's totals, the consumer needs no SyncBN logic
    sync_exchange_block_d<kPrint>(s, const_cast<double*>(acc), n, tid, nthr, sync);
    return;
  }
  const uint32_t epoch = sync_epoch(s);
  for (int i = tid; i < n; i += nthr) sync_push_value_d(s, epoch, i, __ldcg(acc + i));
  sync_publish(s, epoch, tid, sync);
}

// consumer: world total of element idx, added in rank order (bit-identical on every rank)
__device__ __forceinline__ float sync_total(const SyncDesc& s, uint32_t epoch, int idx) {
  const float* my = reinterpret_cast<const float*>(s.peers[s.rank]) + (size_t)(epoch & 1u) * s.world * s.n_max + idx;
  float t = 0.f;
  for (int p = 0; p < s.world; ++p) t += __ldcv(my + (size_t)p * s.n_max);
  return t;
}
__device__ __forceinline__ void sync_total8(const SyncDesc& s, uint32_t epoch, int idx, float* out8) {
  const float* my = reinterpret_cast<const float*>(s.peers[s.rank]) + (size_t)(epoch & 1u) * s.world * s.n_max + idx;
#pragma unroll
  for (int j = 0; j < 8; ++j) out8[j] = 0.f;
  for (int p = 0; p < s.world; ++p) {
    const float4 a = __ldcv(reinterpret_cast<const float4*>(my + (size_t)p * s.n_max));
    const float4 b = __ldcv(reinterpret_cast<const float4*>(my + (size_t)p * s.n_max + 4));
    out8[0] += a.x; out8[1] += a.y; out8[2] += a.z; out8[3] += a.w;
    out8[4] += b.x; out8[5] += b.y; out8[6] += b.z; out8[7] += b.w;
  }
}

// ---- mode 1: the whole exchange inside the producer's last block -----------------------------------------------------------------
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
// fp32 variant (BatchNorm backward sums)
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

// consumer: all threads of the block call this; returns after every rank's flag shows `epoch`
__device__ __forceinline__ void sync_wait_world(const SyncDesc& s, uint32_t epoch) {
  if ((int)threadIdx.x < s.world) {
    const uint32_t* mine = reinterpret_cast<const uint32_t*>(reinterpret_cast<const char*>(s.peers[s.rank]) + sync_flags_offset(s.world, s.n_max)) +
                           (size_t)(epoch & 1u) * s.world + threadIdx.x;
    const long long limit = s.timeout_clocks > 0 ? s.timeout_clocks : (1ll << 62);
    const long long t0 = clock64();
    while (sync_ld_acquire_sys(mine) != epoch) {
      if (clock64() - t0 > limit) {
        printf("seg_b200: SyncBN exchange timeout (rank %d waiting for rank %d, epoch %u; raise SEG_SYNC_TIMEOUT_S)\n", s.rank,
               (int)threadIdx.x, epoch);
        __trap();
      }
    }
  }
  __syncthreads();
}

// consumer, at the very end of the kernel (every thread of every block calls it): the last block to get here advances seq.
// `done` = a zeroed uint32 owned by this launch.
__device__ __forceinline__ void sync_consumer_done(const SyncDesc& s, uint32_t epoch, unsigned* done, unsigned nblocks) {
  __syncthreads();  // every thread of this block has read its totals
  if (threadIdx.x == 0) {
    __threadfence();
    if (atomicAdd(done, 1u) == nblocks - 1u) {
      uint32_t* seq = reinterpret_cast<uint32_t*>(reinterpret_cast<char*>(s.peers[s.rank]) + sync_seq_offset(s.world, s.n_max));
      *seq = epoch;
      __threadfence();
    }
  }
}

}  // namespace seg
