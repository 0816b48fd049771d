// blance_b200/csrc/sticky_rank.cuh — the outcome byte of a step the speculative pass accepted as sticky.
//
// Such a step keeps its k current nodes, in (score, position) order.  A scout packs the rank of current node q
// (0 = best) into bits 2q..2q+1 (srank_pack), the leader stores 0x80 | those bits as one byte per step
// (srank_byte), and k_scatter_stream writes node q to output slot rank(q) (srank_expand).  Bit 7 is the
// "accepted" flag, so only three ranks fit next to it: with k = 4 the rank of node 3 is not packed but derived,
// since the ranks are a permutation of 0..k-1 and sum to k(k-1)/2.  tests/test_sticky_rank_codec.py checks every
// permutation for k = 1..4.  (Host and device: the test compiles this header into a host program.)
#pragma once

#include <cstdint>

namespace blance_dev {

#define BL_SRANK_ACCEPTED 0x80u
#ifndef BL_SRANK_PACKED
#define BL_SRANK_PACKED 3   // ranks carried in the byte (the test overrides it to show that packing all 4 is caught)
#endif

// `ranks` with the rank of current node q added (nodes from BL_SRANK_PACKED on are implied)
template <int K>
__host__ __device__ __forceinline__ uint32_t srank_pack(uint32_t ranks, int q, int rank) {
  return q < BL_SRANK_PACKED ? ranks | ((uint32_t)rank << (2 * q)) : ranks;
}

// the stored byte; `ranks` may carry unrelated bits above bit 7
__host__ __device__ __forceinline__ uint8_t srank_byte(uint32_t ranks) {
  return (uint8_t)(BL_SRANK_ACCEPTED | (ranks & 0xFFu));
}

__host__ __device__ __forceinline__ bool srank_accepted(uint32_t b) { return (b & BL_SRANK_ACCEPTED) != 0; }

// rank of current node q, given the sum of the ranks of nodes 0..q-1
template <int K>
__host__ __device__ __forceinline__ int srank_rank(uint32_t b, int q, int below) {
  return q < BL_SRANK_PACKED ? (int)((b >> (2 * q)) & 3u) : K * (K - 1) / 2 - below;
}

// out[rank(q)] = cur[q] for q < K: the step's nodes in (score, position) order
template <int K>
__host__ __device__ __forceinline__ void srank_expand(uint32_t b, const int32_t* cur, int32_t* out) {
  int below = 0;
#pragma unroll
  for (int q = 0; q < K; ++q) {
    const int r = srank_rank<K>(b, q, below);
    below += r;
    out[r] = cur[q];
  }
}

}  // namespace blance_dev
