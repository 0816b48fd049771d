// blance_b200/csrc/node_load.h — the host launchers of libblance_b200_load.so (node_load.cu): each node's load over
// the maps M_0 .. M_R of a rebalance (blance_moves_load, include/blance_b200.h).  Host-only: c_abi.cu includes it
// and libblance_b200.so links the library.  The library is built with hidden visibility and exports only these
// functions, so neither its kernels nor its CUB instantiations can bind to, or be bound from, the main library's.
//
// The caller owns every buffer: it allocates them on the ctx stream, sized by load_scan_bytes / load_event_bytes and
// by the event count load_count leaves in ev_off[P].  Each launcher enqueues on `st`, adds the kernels it launched
// to *launches and returns the first CUDA error (cudaSuccess otherwise).
#pragma once

#include <cuda_runtime.h>

#include <cstddef>
#include <cstdint>

#define BLANCE_LOAD_API __attribute__((visibility("default")))

namespace blance_load {

struct LoadArgs {
  // one instance: a moves handle's beg rows and CSR ops, or one (scenario, count) of a wave with its ops in a table
  // of MO per partition; the round of each op (-1 = never scheduled) is laid out as the ops are
  const int32_t* beg;               // [P] rows, `stride` apart
  const long long* op_off;          // [P + 1] CSR, or NULL: partition p's ops are [p MO, p MO + op_n[p])
  const uint8_t* op_n;              // [P] (table form)
  const int32_t* op_node;
  const uint8_t* op_state;
  const uint8_t* op_kind;
  const int32_t* op_round;
  const int32_t* weight;            // [P], or NULL: every partition weighs 1
  const uint8_t* pflags;            // [P] begMap membership (PF_IN_PREV | PF_IN_ASSIGN) and PF_HAS_WEIGHT, or NULL: every
                                    // partition has its row and, with `weight`, its weight
  int32_t has_part_weights;         // with pflags: weight[p] applies where pflags[p] has PF_HAS_WEIGHT
  long long stride;
  int32_t P, S, SL, NU, MO;
  int32_t slot_off[9];              // [S + 1]
  // results, [S + 1][NU] each (row S: every state)
  long long* node_beg;
  long long* node_end;
  long long* node_peak;
  int32_t* node_peak_round;
  unsigned long long* peak_key;     // ((load + 2^31) << 32) | ~t, the running maximum
  unsigned long long* over_key;     // [1] (overshoot << 32) | ~q
  // the event count per partition and its exclusive scan, [P + 1] each
  long long* ev_count;
  long long* ev_off;
  void* scan_tmp;
  size_t scan_tmp_bytes;
  // the events, [NE] each, and the sort / merge / scan scratch
  unsigned long long *ev_key, *ev_key2, *run_key;
  int32_t *ev_val, *ev_val2, *run_val, *run_sum;
  int* n_runs;
  void* ev_tmp;
  size_t ev_tmp_bytes;
};

// Scratch bytes of the event-count scan over P partitions.
BLANCE_LOAD_API cudaError_t load_scan_bytes(int32_t P, size_t* bytes, cudaStream_t st);
// Scratch bytes of the sort, merge and scan of NE events whose keys use the low 32 + key_bits bits.
BLANCE_LOAD_API cudaError_t load_event_bytes(long long NE, int key_bits, size_t* bytes, cudaStream_t st);
// node_beg (the load on M_0) and the exact event count: ev_off[p] is partition p's first event, ev_off[P] the total.
BLANCE_LOAD_API cudaError_t load_count(const LoadArgs& A, int sm_count, cudaStream_t st, long long* launches);
// Emits the NE events, merges them per (node, state, t), scans them per (node, state) and takes each key's peak;
// fills node_end, node_peak, node_peak_round and over_key.  Waits for the stream once (the number of merged runs).
BLANCE_LOAD_API cudaError_t load_peaks(const LoadArgs& A, long long NE, int key_bits, int sm_count, cudaStream_t st,
                                       long long* launches);

}  // namespace blance_load
