"""The CPU reference of blance_plan_scenarios_exposure (include/blance_b200.h): the exposure of one (scenario, count)
pair, built from oracles already in the tree - the scenario's next rows (the CPU plan oracle or the device), its
begMap moves (oracle/fast.c CalcPartitionMoves), their lock-step schedule (tests/schedule_oracle.c) and an exposure
oracle of tests/exposure_oracle.py over begMap's partitions, scattered back to all partitions."""
import numpy as np

import exposure_oracle as EO
import schedule_oracle as SO
from test_exposure_oracle import calc_moves

PART_FILL = (("part_min_copies", -1, np.int32), ("part_no_top", 0, np.int32), ("part_flags", 0, np.uint8))


def begmap_rows(t, next_rows):
    """(member [P] bool, beg, end) of scenario tables t: begMap is part_in_prev || part_in_assign; beg is the prev row
    (empty when absent from prevMap), end the next row of an assigned partition and the beg row otherwise."""
    P, SL = t.n_parts, t.n_slots
    in_prev, assigned = np.asarray(t.part_in_prev) != 0, np.asarray(t.part_in_assign) != 0
    member = in_prev | assigned
    beg = np.where(in_prev[:, None], np.asarray(t.prev_rows).reshape(P, SL), -1).astype(np.int32)
    end = np.where(assigned[:, None], np.asarray(next_rows).reshape(P, SL), beg).astype(np.int32)
    return member, np.ascontiguousarray(beg[member]), np.ascontiguousarray(end[member])


def scenario_exposure(t, next_rows, favor_min_nodes, count, node_has_mover=None, domain_parent=None, oracle=EO.vectorised):
    """(exposure dict as moves_exposure returns it, schedule scalars) of scenario tables t (its own constraints,
    the base's top_state) at MaxConcurrentPartitionMovesPerNode `count`; node_has_mover None = the ids < n_nodes."""
    member, beg, end = begmap_rows(t, next_rows)
    slot_off = np.asarray(t.state_slot_off, np.int32)
    off, node, state, kind = calc_moves(slot_off, beg, end, favor_min_nodes)
    NU = t.n_node_ids
    mover = (np.arange(NU) < t.n_nodes).astype(np.uint8) if node_has_mover is None else np.asarray(node_has_mover, np.uint8)
    ro, so, sc = SO.schedule(off, node, kind, NU, max(1, int(count)), mover)
    cons = np.asarray(t.state_constraints, np.int32)
    got = oracle(slot_off, beg, off, node, state, kind, ro, so, cons, int(t.top_state), NU, domain_parent)
    for k, fill, dt in PART_FILL:
        full = np.full(t.n_parts, fill, dt)
        full[member] = got[k]
        got[k] = full
    return got, sc
