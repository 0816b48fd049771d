"""The serial schedule oracle (tests/schedule_oracle.c, TEST INFRASTRUCTURE) and a direct Python reading of the Go
statements it restates.  The C file is compiled on first use into a temporary directory keyed by its contents, so
the source tree stays untouched (it may be read-only)."""
import ctypes
import hashlib
import os
import subprocess
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "schedule_oracle.c")
_LIB = None

WEIGHT = {0: 3, 1: 4, 2: 1, 3: 2}          # MoveOpWeight by enum blance_op_kind (add, del, promote, demote)


def lib():
    global _LIB
    if _LIB is None:
        digest = hashlib.sha256(open(SRC, "rb").read()).hexdigest()[:16]
        d = os.path.join(tempfile.gettempdir(), "blance_sched_oracle_%d" % os.getuid())
        os.makedirs(d, exist_ok=True)
        so = os.path.join(d, "libsched_oracle_%s.so" % digest)
        if not os.path.exists(so):
            tmp = so + ".%d.tmp" % os.getpid()
            subprocess.run([os.environ.get("CC", "gcc"), "-O2", "-std=c11", "-fPIC", "-shared", SRC, "-o", tmp], check=True)
            os.replace(tmp, so)
        L = ctypes.CDLL(so)
        L.oracle_moves_schedule.argtypes = [ctypes.c_int32, ctypes.c_int32] + [ctypes.c_void_p] * 3 + [ctypes.c_int32] + [ctypes.c_void_p] * 4
        _LIB = L
    return _LIB


def schedule(op_off, op_node, op_kind, n_node_ids, max_concurrent, node_has_mover=None):
    """(round_off, sched_op, {rounds, moves_done, stuck_parts, max_batch}) of the lock-step model."""
    op_off = np.ascontiguousarray(op_off, np.int64)
    op_node = np.ascontiguousarray(op_node, np.int32)
    op_kind = np.ascontiguousarray(op_kind, np.uint8)
    P = len(op_off) - 1
    T = int(op_off[-1])
    ro = np.zeros(T + 2, np.int64)
    so = np.zeros(max(T, 1), np.int64)
    sc = np.zeros(4, np.int64)
    mv = None if node_has_mover is None else np.ascontiguousarray(node_has_mover, np.uint8)
    st = lib().oracle_moves_schedule(P, int(n_node_ids), op_off.ctypes.data, op_node.ctypes.data if T else None,
                                     op_kind.ctypes.data if T else None, int(max_concurrent),
                                     None if mv is None else mv.ctypes.data, ro.ctypes.data, so.ctypes.data, sc.ctypes.data)
    assert st == 0
    R, done = int(sc[0]), int(sc[1])
    return ro[:R + 1], so[:done], dict(rounds=R, moves_done=done, stuck_parts=int(sc[2]), max_batch=int(sc[3]))


def go_reading(op_off, op_node, op_kind, n_node_ids, max_concurrent, node_has_mover=None):
    """orchestrate.go:509-591 (runSupplyMoves), 749-763 (findAvailableMovesUnlocked), 482-504
    (filterNextPlausibleMovesForNode) and 177-186 (LowestWeightPartitionMoveForNode), read statement by statement
    under the lock-step model: partitions walked in ascending index, nodes fed in ascending id, every batch done
    before the next round, moves on nodes without a mover never fed.  Returns the batches of every round as
    [[(node, [global op index, ...]), ...], ...]."""
    P = len(op_off) - 1
    nxt = [0] * P
    has = (lambda n: 0 <= n < n_node_ids) if node_has_mover is None else (lambda n: 0 <= n < n_node_ids and node_has_mover[n])
    rounds = []
    while True:
        available = {}
        for p in range(P):                                   # for _, nextMoves := range o.mapPartitionToNextMoves
            if nxt[p] < op_off[p + 1] - op_off[p]:            # if nextMoves.Next < len(nextMoves.Moves)
                node = int(op_node[op_off[p] + nxt[p]])
                available.setdefault(node, []).append(p)
        fed = [n for n in sorted(available) if has(n)]      # a node without a mover is never fed
        if not fed:
            return rounds
        batches = []
        for node in fed:
            arr = list(available[node])
            count = max_concurrent if max_concurrent > 0 else 1
            count = min(count, len(arr))
            picks = []
            while count > 0:
                r = 0
                for i in range(len(arr)):
                    if WEIGHT[int(op_kind[op_off[arr[r]] + nxt[arr[r]]])] > WEIGHT[int(op_kind[op_off[arr[i]] + nxt[arr[i]]])]:
                        r = i
                picks.append(arr[r])
                count -= 1
                arr[r] = arr[-1]
                arr.pop()
            batches.append((node, [int(op_off[p] + nxt[p]) for p in picks]))
            for p in picks:
                nxt[p] += 1
        rounds.append(batches)


def flatten(rounds):
    """round_off / sched_op of go_reading's batches."""
    ro, so = [0], []
    for batches in rounds:
        for _, ops in batches:
            so += ops
        ro.append(len(so))
    return np.asarray(ro, np.int64), np.asarray(so, np.int64)
