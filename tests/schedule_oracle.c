/* tests/schedule_oracle.c — TEST INFRASTRUCTURE, NOT PRODUCT CODE.
 *
 * The lock-step schedule of include/blance_b200.h (blance_moves_schedule) restated serially over the CSR move
 * lists of blance_moves_fetch: an active list in ascending partition index, per-node lists built by an ascending
 * walk (findAvailableMovesUnlocked, orchestrate.go:749-763), then, per node in ascending id, the literal pick and
 * swap-remove loop of filterNextPlausibleMovesForNode (orchestrate.go:482-504) with
 * LowestWeightPartitionMoveForNode (orchestrate.go:177-186).  Each round costs O(active + n_node_ids), so the
 * headline cluster's move lists are checked in seconds.  Built on demand by tests/schedule_oracle.py.
 */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#define SO_EXPORT __attribute__((visibility("default")))

static int op_weight(uint8_t kind) {            /* MoveOpWeight; enum blance_op_kind = add, del, promote, demote */
  static const int w[4] = {3, 4, 1, 2};
  return w[kind & 3];
}

/* Same shape as blance_moves_schedule + blance_moves_schedule_fetch.  round_off: [total_ops + 2]; sched_op:
 * [total_ops]; scalars: rounds, moves_done, stuck_parts, max_batch.  Returns 0, or -5 when out of memory. */
SO_EXPORT int oracle_moves_schedule(int32_t n_parts, int32_t n_node_ids, const int64_t* op_off, const int32_t* op_node,
                                    const uint8_t* op_kind, int32_t max_concurrent_per_node,
                                    const uint8_t* node_has_mover, int64_t* round_off, int64_t* sched_op,
                                    int64_t* scalars) {
  const int32_t count = max_concurrent_per_node <= 0 ? 1 : max_concurrent_per_node;
  int32_t* cur = calloc((size_t)n_parts + 1, sizeof(int32_t));
  int32_t* act = malloc(sizeof(int32_t) * ((size_t)n_parts + 1));
  int32_t* lst = malloc(sizeof(int32_t) * ((size_t)n_parts + 1));
  int32_t* noff = malloc(sizeof(int32_t) * ((size_t)n_node_ids + 2));
  int32_t* fill = malloc(sizeof(int32_t) * ((size_t)n_node_ids + 2));
  if (!cur || !act || !lst || !noff || !fill) { free(cur); free(act); free(lst); free(noff); free(fill); return -5; }
#define PICKABLE(n) ((n) >= 0 && (n) < n_node_ids && (!node_has_mover || node_has_mover[(n)]))
  int64_t stuck = 0, done = 0;
  int32_t A = 0, rounds = 0, max_batch = 0;
  for (int32_t p = 0; p < n_parts; p++) {
    if (op_off[p] == op_off[p + 1]) continue;
    if (PICKABLE(op_node[op_off[p]])) act[A++] = p;
    else stuck++;
  }
  round_off[0] = 0;
  while (A > 0) {
    /* findAvailableMovesUnlocked: partitions appended to their node's list in ascending index */
    memset(noff, 0, sizeof(int32_t) * ((size_t)n_node_ids + 1));
    for (int32_t i = 0; i < A; i++) noff[op_node[op_off[act[i]] + cur[act[i]]] + 1]++;
    for (int32_t n = 0; n < n_node_ids; n++) noff[n + 1] += noff[n];
    memcpy(fill, noff, sizeof(int32_t) * ((size_t)n_node_ids + 1));
    for (int32_t i = 0; i < A; i++) lst[fill[op_node[op_off[act[i]] + cur[act[i]]]]++] = act[i];
    /* filterNextPlausibleMovesForNode per node, ascending node id */
    for (int32_t n = 0; n < n_node_ids; n++) {
      int32_t* arr = lst + noff[n];
      int32_t len = noff[n + 1] - noff[n];
      if (len == 0) continue;
      int32_t c = count > len ? len : count;
      if (c > max_batch) max_batch = c;
      for (; c > 0; c--) {
        int32_t r = 0;                          /* LowestWeightPartitionMoveForNode */
        for (int32_t i = 0; i < len; i++)
          if (op_weight(op_kind[op_off[arr[r]] + cur[arr[r]]]) > op_weight(op_kind[op_off[arr[i]] + cur[arr[i]]])) r = i;
        const int32_t p = arr[r];
        sched_op[done++] = op_off[p] + cur[p];
        cur[p]++;                               /* the batch completes before the next round */
        arr[r] = arr[len - 1];
        len--;
      }
    }
    round_off[++rounds] = done;
    /* drop finished partitions and those whose next move's node has no mover, keeping the order */
    int32_t a2 = 0;
    for (int32_t i = 0; i < A; i++) {
      const int32_t p = act[i];
      if (op_off[p] + cur[p] >= op_off[p + 1]) continue;
      if (PICKABLE(op_node[op_off[p] + cur[p]])) act[a2++] = p;
      else stuck++;
    }
    A = a2;
  }
#undef PICKABLE
  scalars[0] = rounds;
  scalars[1] = done;
  scalars[2] = stuck;
  scalars[3] = max_batch;
  free(cur); free(act); free(lst); free(noff); free(fill);
  return 0;
}
