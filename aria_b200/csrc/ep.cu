// Expert-parallel exchange over NVLink peer memory (no NCCL, no host sync): every rank owns an arena that all peers map
// (aria_b200/peer.py); the kernels below store straight into the peers' arenas through NVSwitch.
//
//   peer_barrier   device-side all-ranks barrier on flags in the arenas (release/acquire at system scope)
//   ep_dispatch    FUSED permute + dispatch: gathers token rows in expert order and stores them directly into the owning
//                  rank's fixed-capacity receive regions, and publishes each block's (count, first sorted row) to the owner
// The way back needs no kernel here: the fc2 grouped GEMM's epilogue stores into the source ranks' buffers (csrc/gemm.cu).
// Replaces the all-to-all of Megatron's dispatcher that the reference stripped out (aria/model/moe_lm.py:296-297).
#include "common.cuh"
#include "ptx.cuh"

namespace aria {

// The epoch lives in device memory and is advanced by the kernel itself, so a CUDA graph that captured the barrier replays
// correctly (every rank executes the same sequence of barriers, so the counters stay in step).
__global__ void peer_barrier_kernel(const uint64_t* __restrict__ peer_flags, int rank, int W, int32_t* __restrict__ epoch_dev) {
  __shared__ int s_epoch;
  if (threadIdx.x == 0) s_epoch = ++(*epoch_dev);
  __syncthreads();
  const int epoch = s_epoch;
  const int s = threadIdx.x;
  if (s >= W) return;
  __threadfence_system();  // everything this GPU stored before the barrier is visible before the flag
  int32_t* remote = reinterpret_cast<int32_t*>(peer_flags[s]) + rank;
  asm volatile("st.release.sys.global.s32 [%0], %1;" ::"l"(remote), "r"(epoch) : "memory");
  const int32_t* mine = reinterpret_cast<const int32_t*>(peer_flags[rank]) + s;
  const long long t0 = clock64();
  int v;
  do {
    asm volatile("ld.acquire.sys.global.s32 %0, [%1];" : "=r"(v) : "l"(mine) : "memory");
    if (clock64() - t0 > 80000000000ll) {  // ~40 s: ranks can be seconds apart at the first barrier (lazy module loads), never minutes
      printf("aria_b200: peer barrier timeout (rank %d waiting for %d, epoch %d, saw %d)\n", rank, s, epoch, v);
      __trap();
    }
  } while (v < epoch);
}

// ---------------------------------------------------------------------------------------------------------------------
// Fused exchange (round 2).  Every owner rank p keeps, per (local expert el, source rank s) - region index el * W + s, so that the
// W regions that are multiplied by the same expert's weights are neighbours in the grouped GEMM's tile order and the weights are
// read from HBM once (cfg 2: the expert GEMMs are weight-streaming bound) - a FIXED-CAPACITY region of `cap`
// rows in its receive buffer (a token picks an expert at most once, so cap = T_max bounds it): a sender needs nobody else's
// counts to know where its rows go.  ep_dispatch gathers the token rows in expert order and stores each straight into the
// owner's region over NVLink (fused permute + dispatch), and publishes (count, first sorted row) of each of its blocks into
// the owner's meta arrays.  After ONE device-side barrier the owner runs its grouped GEMMs directly on the regions
// (aria_gemm group_counts) and the fc2 epilogue stores every output row straight into the source rank's combine buffer
// (aria_gemm out_group_base / out_group_row0): the return all-to-all is the GEMM's epilogue.  Two barriers per layer, no
// counts exchange, no layout kernel, no copy kernel on the way back.
__global__ void __launch_bounds__(256) ep_dispatch_kernel(const uint4* __restrict__ x, const int32_t* __restrict__ src_token,
                                                          const int32_t* __restrict__ offsets, const uint64_t* __restrict__ peer_recv,
                                                          const uint64_t* __restrict__ peer_counts, const uint64_t* __restrict__ peer_row0,
                                                          int rank, int E, int E_loc, int cap, int vec_per_row) {
  const int W = E / E_loc;
  __shared__ int s_off[1025];
  for (int i = threadIdx.x; i <= E; i += blockDim.x) s_off[i] = offsets[i];
  __syncthreads();
  if (blockIdx.x == 0) {  // meta: my block for global expert e = group (rank, e % E_loc) of owner e / E_loc
    for (int e = threadIdx.x; e < E; e += blockDim.x) {
      const int p = e / E_loc, g = (e - p * E_loc) * W + rank;
      reinterpret_cast<int32_t*>(peer_counts[p])[g] = s_off[e + 1] - s_off[e];
      reinterpret_cast<int32_t*>(peer_row0[p])[g] = s_off[e];
    }
  }
  const int total = s_off[E];
  const int lane = threadIdx.x & 31, wpb = blockDim.x >> 5;
  for (int r = blockIdx.x * wpb + (threadIdx.x >> 5); r < total; r += gridDim.x * wpb) {
    int lo = 0, hi = E;  // expert of sorted row r: last e with s_off[e] <= r
    while (hi - lo > 1) {
      const int mid = (lo + hi) >> 1;
      if (s_off[mid] <= r) lo = mid; else hi = mid;
    }
    const int e = lo, p = e / E_loc, el = e - p * E_loc;
    uint4* dst = reinterpret_cast<uint4*>(peer_recv[p]) +
                 (static_cast<int64_t>(el * W + rank) * cap + (r - s_off[e])) * vec_per_row;
    const int st = src_token[r];
    if (st < 0) {  // alignment pad row of the training layout: zeros
      for (int v = lane; v < vec_per_row; v += 32) dst[v] = make_uint4(0, 0, 0, 0);
    } else {
      const uint4* src = x + static_cast<int64_t>(st) * vec_per_row;
      for (int v = lane; v < vec_per_row; v += 32) dst[v] = __ldg(src + v);
    }
  }
}

}  // namespace aria

using namespace aria;

extern "C" int aria_ep_dispatch(const void* x, const int32_t* src_token, const int32_t* offsets, const uint64_t* peer_recv,
                                const uint64_t* peer_counts, const uint64_t* peer_row0, int32_t rank, int32_t W, int32_t E,
                                int32_t cap, int32_t d, int64_t max_rows, aria_stream_t stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  ARIA_CHECK_ARG(x && src_token && offsets && peer_recv && peer_counts && peer_row0);
  ARIA_CHECK_ARG(W >= 1 && E >= 1 && E <= 1024 && E % W == 0 && rank >= 0 && rank < W && cap >= 1 && d % 8 == 0 && max_rows >= 0);
  int64_t blocks = (max_rows + 7) / 8;
  const int64_t cap_blocks = static_cast<int64_t>(sm_count()) * 8;
  if (blocks > cap_blocks) blocks = cap_blocks;
  if (blocks < 1) blocks = 1;
  ep_dispatch_kernel<<<static_cast<int>(blocks), 256, 0, stream>>>(static_cast<const uint4*>(x), src_token, offsets, peer_recv,
                                                                   peer_counts, peer_row0, rank, E, E / W, cap, d / 8);
  return check_launch("ep_dispatch_kernel");
}

extern "C" int aria_peer_barrier(const uint64_t* peer_flags, int32_t rank, int32_t W, int32_t* epoch_dev, aria_stream_t stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  ARIA_CHECK_ARG(peer_flags && epoch_dev && W >= 1 && W <= 32 && rank >= 0 && rank < W);
  peer_barrier_kernel<<<1, 32, 0, stream>>>(peer_flags, rank, W, epoch_dev);
  return check_launch("peer_barrier_kernel");
}
