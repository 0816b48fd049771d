// integration/blance_b200.go — the cgo binding a blance maintainer adds to the package
// (drop it next to api.go and rename the bodies as INTEGRATION.md says).
//
// UNTESTED GO: this image has no Go toolchain.  The file is a transliteration of
// blance_b200/csrc/host_api.cpp (InternPlan / UninternPlan / ReplayCallerMutation /
// intern_moves), which is the tested implementation of the same logic: the parity tests
// of this repo go through that C++ twin.  It is written against the unmodified types and
// helpers of the reference package (api.go, plan.go, misc.go, moves.go).
//
//   PlanNextMapEx       api.go:147-157  ->  planNextMapExB200      ->  blance_plan_next_map
//   CalcPartitionMoves  moves.go:41-119 ->  calcPartitionMovesB200 ->  blance_calc_partition_moves
//
// Inside libblance_b200 there is no CPU fallback.  This shim lives in the same package as the Go planner, so the
// inputs the device path reports as BLANCE_ERR_UNSUPPORTED (more than 8 states, 32 slots, 8192 nodes, 16
// constraints; a CustomNodeSorter; Partition.Name != key ...) and a missing / failed device (BLANCE_ERR_CUDA) go
// to the package's own planNextMapEx / calcPartitionMovesGo - a drop-in must not turn valid inputs into panics.
// BLANCE_ERR_INVALID_ARG still panics: the reference panics (or misbehaves) on those inputs too.

//go:build cgo

package blance

/*
#cgo LDFLAGS: -lblance_b200
#include <stdlib.h>
#include <string.h>
#include "blance_b200.h"
*/
import "C"

import (
	"fmt"
	"reflect"
	"sort"
	"strconv"
	"sync"
	"unsafe"
)

var (
	b200Once sync.Once
	b200Ctx  *C.blance_ctx
)

// b200CheckTables makes every plan run blance_plan_in_check on its tables first (set it in the shim's own tests).
var b200CheckTables = false

func b200() *C.blance_ctx {
	b200Once.Do(func() {
		if st := C.blance_ctx_create(&b200Ctx, -1); st != C.BLANCE_OK {
			panic("blance_b200: " + C.GoString(C.blance_last_error(nil)))
		}
	})
	return b200Ctx
}

// cArena owns the C-side arrays of one call (cgo: no Go pointers to Go pointers may cross,
// so every table lives in C memory for the duration of the call).
type cArena struct{ ptrs []unsafe.Pointer }

func (a *cArena) free() {
	for _, p := range a.ptrs {
		C.free(p)
	}
}
func (a *cArena) i32(n int, fill int32) (*C.int32_t, []int32) {
	p := C.malloc(C.size_t(4 * (n + 1)))
	a.ptrs = append(a.ptrs, p)
	s := unsafe.Slice((*int32)(p), n+1)
	for i := range s {
		s[i] = fill
	}
	return (*C.int32_t)(p), s[:n]
}
func (a *cArena) u8(n int) (*C.uint8_t, []uint8) {
	p := C.calloc(C.size_t(n+1), 1)
	a.ptrs = append(a.ptrs, p)
	return (*C.uint8_t)(p), unsafe.Slice((*uint8)(p), n+1)[:n]
}
func (a *cArena) u32(n int) (*C.uint32_t, []uint32) {
	p := C.calloc(C.size_t(n+1), 4)
	a.ptrs = append(a.ptrs, p)
	return (*C.uint32_t)(p), unsafe.Slice((*uint32)(p), n+1)[:n]
}

// interner: node names -> dense ids; nodesAll first (ids = positions, plan.go:72-75), then
// any other name that occurs in rows or in nodesToRemove / nodesToAdd (never candidates).
type interner struct {
	ids   map[string]int32
	names []string
}

func (it *interner) get(s string) int32 {
	if id, ok := it.ids[s]; ok {
		return id
	}
	id := int32(len(it.names))
	it.ids[s] = id
	it.names = append(it.names, s)
	return id
}

// partitionOrder: keys(prevMap) U keys(partitionsToAssign) in the name order of the
// partition sort key (plan.go:519-528, 512): "%10d" of the name when it is a non-negative
// integer, else the name; ties by the raw name.
func partitionOrder(prevMap, partitionsToAssign PartitionMap) []string {
	type nameKey struct {
		numeric bool
		v       int64
		padded  string
		raw     string
	}
	seen := make(map[string]struct{}, len(prevMap)+len(partitionsToAssign))
	keys := make([]nameKey, 0, len(prevMap)+len(partitionsToAssign))
	add := func(m PartitionMap) {
		for name := range m {
			if _, dup := seen[name]; dup {
				continue
			}
			seen[name] = struct{}{}
			k := nameKey{raw: name, padded: name}
			if v, err := strconv.Atoi(name); err == nil && v >= 0 {
				k.padded = fmt.Sprintf("%10d", v)
				// ten-character padded forms order like the numbers: compare as integers
				k.numeric, k.v = v < 10000000000, int64(v)
			}
			keys = append(keys, k)
		}
	}
	add(prevMap)
	add(partitionsToAssign)
	sort.Slice(keys, func(i, j int) bool {
		a, b := &keys[i], &keys[j]
		if a.numeric && b.numeric {
			if a.v != b.v {
				return a.v < b.v
			}
			return a.raw < b.raw
		}
		if a.padded != b.padded {
			return a.padded < b.padded
		}
		return a.raw < b.raw
	})
	out := make([]string, len(keys))
	for i := range keys {
		out[i] = keys[i].raw
	}
	return out
}

// planNextMapExB200 replaces plan.go:23-58.  Same signature, same results, same mutation of
// the caller's maps.
func planNextMapExB200(prevMap, partitionsToAssign PartitionMap,
	nodesAll, nodesToRemove, nodesToAdd []string,
	model PartitionModel, opts PlanNextMapOptions) (PartitionMap, map[string][]string) {

	// plan.go:580: an application that replaced the sorter keeps the Go planner (func values only compare
	// through reflect)
	if reflect.ValueOf(CustomNodeSorter).Pointer() != reflect.ValueOf(defaultNodeSorter).Pointer() {
		// a func value cannot cross the C ABI (BLANCE_ERR_UNSUPPORTED): the Go planner keeps this call
		return planNextMapEx(prevMap, partitionsToAssign, nodesAll, nodesToRemove, nodesToAdd, model, opts)
	}
	var ar cArena
	defer ar.free()

	// ---- nodes
	nodes := &interner{ids: map[string]int32{}}
	for _, n := range nodesAll {
		if _, dup := nodes.ids[n]; dup {
			panic("blance_b200: nodesAll contains '" + n + "' twice")
		}
		nodes.get(n)
	}
	N := len(nodesAll)

	// ---- states in sortStateNames order (plan.go:437-447), constraints after the override
	states := sortStateNames(model)
	S := len(states)
	stateID := make(map[string]int, S)
	for i, s := range states {
		stateID[s] = i
	}
	pPrio, prio := ar.i32(S, 0)
	pCons, cons := ar.i32(S, 0)
	pStick, stick := ar.i32(S, 0)
	pHasStick, hasStick := ar.u8(S)
	topState := -1
	for i, s := range states {
		prio[i] = int32(model[s].Priority)
		k := model[s].Constraints
		if opts.ModelStateConstraints != nil { // plan.go:308-319
			if v, ok := opts.ModelStateConstraints[s]; ok {
				k = v
			}
		}
		cons[i] = int32(k)
		if opts.StateStickiness != nil {
			if v, ok := opts.StateStickiness[s]; ok {
				stick[i], hasStick[i] = int32(v), 1
			}
		}
	}
	byName := append([]string(nil), states...)
	sort.Strings(byName)
	for _, s := range byName { // plan.go:126-132 (map order in the reference; first by name here)
		if topState < 0 || model[s].Priority < int(prio[topState]) {
			topState = stateID[s]
		}
	}

	// ---- partitions
	partNames := partitionOrder(prevMap, partitionsToAssign)
	PU := len(partNames)
	partID := make(map[string]int, PU)
	for i, n := range partNames {
		partID[n] = i
	}

	// ---- slot layout: a state's range holds max(constraints, longest input list)
	capS := make([]int, S)
	for i := range capS {
		if cons[i] > 0 {
			capS[i] = int(cons[i])
		}
	}
	scan := func(m PartitionMap, mustBeModel bool) {
		for name, p := range m {
			for sn, list := range p.NodesByState {
				s, ok := stateID[sn]
				if !ok {
					if mustBeModel {
						panic("blance_b200: partition '" + name + "' has state '" + sn + "' that is not in the model") // plan.go:148
					}
					continue
				}
				if len(list) > capS[s] {
					capS[s] = len(list)
				}
			}
		}
	}
	scan(prevMap, false)
	scan(partitionsToAssign, true)
	pOff, off := ar.i32(S+1, 0)
	for i := 0; i < S; i++ {
		off[i+1] = off[i] + int32(capS[i])
	}
	SL := int(off[S])

	// ---- rows, shapes, weights
	pInPrev, inPrev := ar.u8(PU)
	pInAssign, inAssign := ar.u8(PU)
	pPrevRows, prevRows := ar.i32(PU*SL, C.BLANCE_NO_NODE)
	pCurRows, curRows := ar.i32(PU*SL, C.BLANCE_NO_NODE)
	pPrevShape, prevShape := ar.u8(PU * S) // BLANCE_SHAPE_ABSENT = 0
	pCurShape, curShape := ar.u8(PU * S)
	pWeight, weight := ar.i32(PU, 1)
	pHasWeight, hasWeight := ar.u8(PU)
	pRank, rank := ar.i32(PU, 0)
	for i := range rank {
		rank[i] = int32(i)
	}
	if opts.PartitionWeights != nil {
		for name, w := range opts.PartitionWeights {
			if p, ok := partID[name]; ok {
				weight[p], hasWeight[p] = int32(w), 1
			}
		}
	}
	type extra struct{ part, node int32 }
	var extras []extra // prevMap entries under non-model states: they only feed the totals (plan.go:118-124)
	fill := func(m PartitionMap, rows []int32, shape []uint8, present []uint8, isPrev bool) {
		for name, p := range m {
			pi := partID[name]
			present[pi] |= 1
			for sn, list := range p.NodesByState {
				s, ok := stateID[sn]
				if !ok {
					if isPrev {
						present[pi] = 3 // bit 1: a key outside the model, reflect.DeepEqual never matches it (plan.go:38)
						for _, n := range list {
							extras = append(extras, extra{int32(pi), nodes.get(n)})
						}
					}
					continue
				}
				if list == nil {
					shape[pi*S+s] = C.BLANCE_SHAPE_NIL
				} else {
					shape[pi*S+s] = C.BLANCE_SHAPE_LIST
				}
				slot := int(off[s])
				for _, n := range list {
					rows[pi*SL+slot] = nodes.get(n)
					slot++
				}
			}
		}
	}
	fill(prevMap, prevRows, prevShape, inPrev, true)
	fill(partitionsToAssign, curRows, curShape, inAssign, false)

	// ---- node flags (after every name that can occur has an id)
	for _, n := range nodesToRemove {
		nodes.get(n)
	}
	for _, n := range nodesToAdd {
		nodes.get(n)
	}
	NU := len(nodes.names)
	pRemoved, removed := ar.u8(NU)
	pAdded, added := ar.u8(NU)
	for _, n := range nodesToRemove {
		removed[nodes.ids[n]] = 1
	}
	for _, n := range nodesToAdd {
		added[nodes.ids[n]] = 1
	}
	pNodeW, nodeW := ar.i32(N, 0)
	pHasNodeW, hasNodeW := ar.u8(N)
	if opts.NodeWeights != nil {
		for n, w := range opts.NodeWeights {
			if id, ok := nodes.ids[n]; ok && int(id) < N {
				nodeW[id], hasNodeW[id] = int32(w), 1
			}
		}
	}
	if len(nodesToRemove) > 0 { // plan.go:544-545 dereferences prevMap[name]
		for p := 0; p < PU; p++ {
			if inAssign[p] == 1 && inPrev[p] == 0 {
				panic("blance_b200: partition '" + partNames[p] + "' is being assigned with nodesToRemove set but is missing from prevMap")
			}
		}
	}
	pExtraFirst, extraFirst := ar.i32(N, 0)
	pExtraRest, extraRest := ar.i32(N, 0)
	for _, e := range extras {
		if int(e.node) >= N {
			continue
		}
		w := int32(1)
		if opts.PartitionWeights != nil && hasWeight[e.part] == 1 {
			w = weight[e.part]
		}
		extraFirst[e.node] += w
		if inAssign[e.part] == 0 {
			extraRest[e.node] += w
		}
	}

	// ---- hierarchy bit sets, with the reference's own helpers (plan.go:703-774)
	pRuleOff, ruleOff := ar.i32(S+1, 0)
	var rules []*HierarchyRule
	if opts.HierarchyRules != nil {
		for i, s := range states {
			rules = append(rules, opts.HierarchyRules[s]...)
			ruleOff[i+1] = int32(len(rules))
		}
	}
	nHierBits := N
	var pMask *C.uint32_t
	if len(rules) > 0 {
		children := mapParentsToMapChildren(opts.NodeHierarchy)
		extraBits := &interner{ids: map[string]int32{}}
		lists := make([][]int32, len(rules)*(NU+1))
		for r, rule := range rules {
			for a := 0; a <= NU; a++ {
				anchor := ""
				if a < NU {
					anchor = nodes.names[a]
				}
				for _, leaf := range includeExcludeNodes(anchor, rule.IncludeLevel, rule.ExcludeLevel,
					opts.NodeHierarchy, children) {
					if id, ok := nodes.ids[leaf]; ok && int(id) < N {
						lists[r*(NU+1)+a] = append(lists[r*(NU+1)+a], id)
					} else {
						lists[r*(NU+1)+a] = append(lists[r*(NU+1)+a], int32(N)+extraBits.get(leaf))
					}
				}
			}
		}
		nHierBits = N + len(extraBits.names)
		HW := (nHierBits + 31) / 32
		var mask []uint32
		pMask, mask = ar.u32(len(lists) * HW)
		for i, l := range lists {
			for _, b := range l {
				mask[i*HW+int(b>>5)] |= 1 << uint(b&31)
			}
		}
	}

	// ---- the call
	var in C.blance_plan_in
	in.n_nodes, in.n_node_ids, in.n_states = C.int32_t(N), C.int32_t(NU), C.int32_t(S)
	in.n_parts, in.n_slots = C.int32_t(PU), C.int32_t(SL)
	in.max_iters = C.int32_t(MaxIterationsPerPlan)
	if topState >= 0 {
		in.top_state = C.int32_t(topState)
	}
	if NodeScoreBooster != nil {
		in.booster_kind = C.BLANCE_BOOSTER_CBGT_MAX // the only booster that can cross the ABI (control_test.go:19-26)
	}
	b2i := func(b bool) C.int32_t {
		if b {
			return 1
		}
		return 0
	}
	in.add_is_nil = b2i(nodesToAdd == nil)
	in.has_part_weights = b2i(opts.PartitionWeights != nil)
	in.has_node_weights = b2i(opts.NodeWeights != nil)
	in.has_hier_rules = b2i(opts.HierarchyRules != nil)
	in.state_priority, in.state_constraints, in.state_slot_off = pPrio, pCons, pOff
	in.state_stickiness, in.state_has_stickiness = pStick, pHasStick
	in.node_removed, in.node_added = pRemoved, pAdded
	in.node_weight, in.node_has_weight = pNodeW, pHasNodeW
	in.part_in_prev, in.part_in_assign = pInPrev, pInAssign
	in.part_weight, in.part_has_weight, in.part_name_rank = pWeight, pHasWeight, pRank
	in.prev_rows, in.prev_shape, in.cur_rows, in.cur_shape = pPrevRows, pPrevShape, pCurRows, pCurShape
	in.extra_tot_first, in.extra_tot_rest = pExtraFirst, pExtraRest
	in.n_rules, in.n_hier_bits = C.int32_t(len(rules)), C.int32_t(nHierBits)
	in.rule_off, in.ie_mask = pRuleOff, pMask

	var out C.blance_plan_out
	pNext, next := ar.i32(PU*SL, C.BLANCE_NO_NODE)
	pNextShape, nextShape := ar.u8(PU * S)
	pWarn, warn := ar.u8(PU * S)
	out.next_rows, out.next_shape, out.warn = pNext, pNextShape, pWarn

	if b200CheckTables { // development aid: the planning call itself does not scan every cell
		var msg [256]C.char
		if st := C.blance_plan_in_check(&in, &msg[0], 256); st == C.BLANCE_ERR_UNSUPPORTED {
			return planNextMapEx(prevMap, partitionsToAssign, nodesAll, nodesToRemove, nodesToAdd, model, opts)
		} else if st != C.BLANCE_OK {
			panic("blance_b200: malformed tables: " + C.GoString(&msg[0]))
		}
	}
	if st := C.blance_plan_next_map(b200(), &in, &out); st != C.BLANCE_OK {
		if st == C.BLANCE_ERR_UNSUPPORTED || st == C.BLANCE_ERR_CUDA || st == C.BLANCE_ERR_NOMEM {
			// nothing was mutated yet: the Go planner answers (same results, only slower)
			return planNextMapEx(prevMap, partitionsToAssign, nodesAll, nodesToRemove, nodesToAdd, model, opts)
		}
		panic("blance_b200: " + C.GoString(C.blance_last_error(b200())))
	}
	if out.iters_run <= 0 { // MaxIterationsPerPlan <= 0: plan.go:32,57
		return nil, nil
	}

	// ---- rows -> PartitionMap (plan.go:326-330), warnings (plan.go:231-234)
	nextMap := PartitionMap{}
	warnings := map[string][]string{}
	for p := 0; p < PU; p++ {
		if inAssign[p] == 0 {
			continue
		}
		part := &Partition{Name: partNames[p], NodesByState: map[string][]string{}}
		for s := 0; s < S; s++ {
			switch nextShape[p*S+s] {
			case C.BLANCE_SHAPE_ABSENT:
				continue
			case C.BLANCE_SHAPE_NIL:
				part.NodesByState[states[s]] = nil
			default:
				list := []string{}
				for i := int(off[s]); i < int(off[s+1]) && next[p*SL+i] != C.BLANCE_NO_NODE; i++ {
					list = append(list, nodes.names[next[p*SL+i]])
				}
				part.NodesByState[states[s]] = list
			}
			if warn[p*S+s] == 1 {
				warnings[part.Name] = append(warnings[part.Name],
					fmt.Sprintf("could not meet constraints: %d, stateName: %s, partitionName: %s",
						cons[s], states[s], part.Name))
			}
		}
		nextMap[part.Name] = part
	}

	// plan.go:49-52: the caller's maps hold the new partitions whenever a second iteration ran
	if out.iters_run >= 2 || out.converged == 0 {
		for name, p := range nextMap {
			prevMap[name] = p
			partitionsToAssign[name] = p
		}
	}
	return nextMap, warnings
}

// calcPartitionMovesB200 replaces moves.go:41-119 for one partition (a batch of one; the
// vectorised form passes every partition of a map in one call: op_count[p] ops each).
func calcPartitionMovesB200(states []string, beg, end map[string][]string, favorMinNodes bool) []NodeStateOp {
	var ar cArena
	defer ar.free()
	nodes := &interner{ids: map[string]int32{}}
	// `states` first (they are the ones walked, moves.go:66,92), then any other key of beg / end
	// (they only feed the adds / dels sets, moves.go:60-64), in sorted order for determinism
	names := append([]string(nil), states...)
	known := map[string]bool{}
	for _, s := range states {
		known[s] = true
	}
	var others []string
	for _, m := range []map[string][]string{beg, end} {
		for s := range m {
			if !known[s] {
				known[s] = true
				others = append(others, s)
			}
		}
	}
	sort.Strings(others)
	names = append(names, others...)
	S := len(names)
	pOff, off := ar.i32(S+1, 0)
	for i, s := range names {
		w := len(beg[s])
		if len(end[s]) > w {
			w = len(end[s])
		}
		off[i+1] = off[i] + int32(w)
	}
	SL := int(off[S])
	pBeg, begRows := ar.i32(SL, C.BLANCE_NO_NODE)
	pEnd, endRows := ar.i32(SL, C.BLANCE_NO_NODE)
	for i, s := range names {
		for j, n := range beg[s] {
			begRows[int(off[i])+j] = nodes.get(n)
		}
		for j, n := range end[s] {
			endRows[int(off[i])+j] = nodes.get(n)
		}
	}
	maxOps := 2*SL + 1
	pNode, opNode := ar.i32(maxOps, 0)
	pState, opState := ar.u8(maxOps)
	pKind, opKind := ar.u8(maxOps)
	pCount, opCount := ar.i32(1, 0)
	fav := C.int32_t(0)
	if favorMinNodes {
		fav = 1
	}
	if st := C.blance_calc_partition_moves(b200(), 1, C.int32_t(S), C.int32_t(len(states)), pOff, pBeg, pEnd,
		fav, C.int32_t(maxOps), pNode, pState, pKind, pCount); st != C.BLANCE_OK {
		panic("blance_b200: " + C.GoString(C.blance_last_error(b200())))
	}
	kinds := [...]string{"add", "del", "promote", "demote"}
	var ops []NodeStateOp
	for i := 0; i < int(opCount[0]); i++ {
		st := ""
		if opState[i] != C.BLANCE_OP_STATE_NONE {
			st = names[opState[i]]
		}
		ops = append(ops, NodeStateOp{Node: nodes.names[opNode[i]], State: st, Op: kinds[opKind[i]]})
	}
	return ops
}

// seedNextMovesB200 replaces the loop of orchestrate.go:273-287: CalcPartitionMoves for EVERY partition of
// begMap in one device call (blance_moves_create), returned as the map of *NextMoves the orchestrator keeps.
// One partition at a time (calcPartitionMovesB200 above) costs a launch and a round trip per partition and is
// slower than the Go function it replaces; this batched form is the one to wire in.  The returned handle stays
// valid until blance_moves_free and answers findAvailableMovesUnlocked (orchestrate.go:749-763) and the
// FindMoveFunc's pick (orchestrate.go:177-186) for a vector of cursors with blance_moves_available - see
// availableMovesB200.  UNTESTED GO, like the rest of this file; the C ABI underneath is covered by
// tests/test_gpu_parity.py::test_moves_plan_csr_and_available_moves.
type movesB200 struct {
	h         *C.blance_moves
	partNames []string // partition index -> name (sorted: the fixed order that replaces Go's map order)
	nodeNames []string
	nNodeIDs  int
}

func seedNextMovesB200(states []string, begMap, endMap PartitionMap, favorMinNodes bool) (map[string]*NextMoves, *movesB200) {
	partNames := make([]string, 0, len(begMap))
	for name := range begMap {
		partNames = append(partNames, name)
	}
	sort.Strings(partNames)
	nodes := &interner{ids: map[string]int32{}}
	// slot layout: the visited states first, every list as wide as the longest one of that state
	S := len(states)
	width := make([]int, S)
	for _, name := range partNames {
		for i, s := range states {
			if w := len(begMap[name].NodesByState[s]); w > width[i] {
				width[i] = w
			}
			if e := endMap[name]; e != nil {
				if w := len(e.NodesByState[s]); w > width[i] {
					width[i] = w
				}
			}
		}
	}
	var ar cArena
	defer ar.free()
	pOff, off := ar.i32(S+1, 0)
	for i := range states {
		off[i+1] = off[i] + int32(width[i])
	}
	SL, P := int(off[S]), len(partNames)
	pBeg, begRows := ar.i32(P*SL, C.BLANCE_NO_NODE)
	pEnd, endRows := ar.i32(P*SL, C.BLANCE_NO_NODE)
	for p, name := range partNames {
		for i, s := range states {
			for j, n := range begMap[name].NodesByState[s] {
				begRows[p*SL+int(off[i])+j] = nodes.get(n)
			}
			if e := endMap[name]; e != nil {
				for j, n := range e.NodesByState[s] {
					endRows[p*SL+int(off[i])+j] = nodes.get(n)
				}
			}
		}
	}
	fav := C.int32_t(0)
	if favorMinNodes {
		fav = 1
	}
	m := &movesB200{partNames: partNames, nodeNames: nodes.names, nNodeIDs: len(nodes.names)}
	var total C.int64_t
	if st := C.blance_moves_create(b200(), C.int32_t(P), C.int32_t(S), C.int32_t(S), pOff, pBeg, pEnd, fav,
		C.int32_t(m.nNodeIDs), &m.h, &total); st != C.BLANCE_OK {
		return nil, nil // the caller keeps the Go loop of orchestrate.go:273-287
	}
	opOff := make([]C.int64_t, P+1)
	opNode := make([]C.int32_t, int(total)+1)
	opState := make([]C.uint8_t, int(total)+1)
	opKind := make([]C.uint8_t, int(total)+1)
	if st := C.blance_moves_fetch(b200(), m.h, &opOff[0], &opNode[0], &opState[0], &opKind[0]); st != C.BLANCE_OK {
		C.blance_moves_free(b200(), m.h)
		return nil, nil
	}
	kinds := [...]string{"add", "del", "promote", "demote"}
	out := make(map[string]*NextMoves, P)
	for p, name := range partNames {
		moves := make([]NodeStateOp, 0, int(opOff[p+1]-opOff[p]))
		for k := opOff[p]; k < opOff[p+1]; k++ {
			st := ""
			if opState[k] != C.BLANCE_OP_STATE_NONE {
				st = states[opState[k]]
			}
			moves = append(moves, NodeStateOp{Node: m.nodeNames[opNode[k]], State: st, Op: kinds[opKind[k]]})
		}
		out[name] = &NextMoves{Partition: name, Next: 0, Moves: moves}
	}
	return out, m
}

// availableMovesB200 answers one round of findAvailableMovesUnlocked (orchestrate.go:749-763): for the cursors
// of `next` (partition name -> NextMoves.Next) it returns, per node, the partitions whose next move is on that
// node, and the partition LowestWeightPartitionMoveForNode (orchestrate.go:177-186) would pick there.
func (m *movesB200) availableMovesB200(next map[string]int) (byNode map[string][]string, best map[string]string) {
	P := len(m.partNames)
	cur := make([]C.int32_t, P+1)
	for p, name := range m.partNames {
		cur[p] = C.int32_t(next[name])
	}
	nodeOff := make([]C.int32_t, m.nNodeIDs+1)
	nodeParts := make([]C.int32_t, P+1)
	bestPart := make([]C.int32_t, m.nNodeIDs+1)
	if st := C.blance_moves_available(b200(), m.h, &cur[0], &nodeOff[0], &nodeParts[0], &bestPart[0]); st != C.BLANCE_OK {
		return nil, nil
	}
	byNode, best = map[string][]string{}, map[string]string{}
	for n := 0; n < m.nNodeIDs; n++ {
		for k := nodeOff[n]; k < nodeOff[n+1]; k++ {
			byNode[m.nodeNames[n]] = append(byNode[m.nodeNames[n]], m.partNames[nodeParts[k]])
		}
		if bestPart[n] >= 0 {
			best[m.nodeNames[n]] = m.partNames[bestPart[n]]
		}
	}
	return byNode, best
}

// assignCallB200 holds the arguments of one AssignPartitionsFunc call of a scheduled round.
type assignCallB200 struct {
	Node                      string
	Partitions, States, Ops []string
}

// scheduleB200 computes the whole rebalance the orchestrator would run (orchestrate.go:482-504, 509-591, 749-763,
// 177-186) under the lock-step model of blance_moves_schedule (include/blance_b200.h): rounds[r] lists round r's
// AssignPartitionsFunc calls in node-id order, each in pick order.  A node outside nodesAll has no mover, so a
// partition whose next move is on it never advances.  states must be the list seedNextMovesB200 was given.
// UNTESTED GO; the C ABI underneath is covered by tests/test_schedule_gpu.py.
func (m *movesB200) scheduleB200(maxConcurrent int, nodesAll, states []string) ([][]assignCallB200, error) {
	inAll := map[string]bool{}
	for _, n := range nodesAll {
		inAll[n] = true
	}
	mover := make([]C.uint8_t, m.nNodeIDs+1)
	for i, n := range m.nodeNames {
		if inAll[n] {
			mover[i] = 1
		}
	}
	var so C.blance_schedule_out
	if st := C.blance_moves_schedule(b200(), m.h, C.int32_t(maxConcurrent), &mover[0], &so); st != C.BLANCE_OK {
		return nil, fmt.Errorf("blance_moves_schedule: %d", int(st))
	}
	roundOff := make([]C.int64_t, int(so.rounds)+1)
	sched := make([]C.int64_t, int(so.moves_done)+1)
	if st := C.blance_moves_schedule_fetch(b200(), m.h, &roundOff[0], &sched[0]); st != C.BLANCE_OK {
		return nil, fmt.Errorf("blance_moves_schedule_fetch: %d", int(st))
	}
	P := len(m.partNames)
	opOff := make([]C.int64_t, P+1)
	if st := C.blance_moves_fetch(b200(), m.h, &opOff[0], nil, nil, nil); st != C.BLANCE_OK {
		return nil, fmt.Errorf("blance_moves_fetch: %d", int(st))
	}
	total := int(opOff[P])
	opNode := make([]C.int32_t, total+1)
	opState := make([]C.uint8_t, total+1)
	opKind := make([]C.uint8_t, total+1)
	if st := C.blance_moves_fetch(b200(), m.h, &opOff[0], &opNode[0], &opState[0], &opKind[0]); st != C.BLANCE_OK {
		return nil, fmt.Errorf("blance_moves_fetch: %d", int(st))
	}
	kinds := [...]string{"add", "del", "promote", "demote"}
	rounds := make([][]assignCallB200, int(so.rounds))
	for r := range rounds {
		for i := roundOff[r]; i < roundOff[r+1]; i++ {
			o := sched[i]
			p := sort.Search(P, func(q int) bool { return opOff[q+1] > o })
			node := m.nodeNames[opNode[o]]
			if len(rounds[r]) == 0 || rounds[r][len(rounds[r])-1].Node != node {
				rounds[r] = append(rounds[r], assignCallB200{Node: node})
			}
			c := &rounds[r][len(rounds[r])-1]
			st := ""
			if opState[o] != C.BLANCE_OP_STATE_NONE {
				st = states[opState[o]]
			}
			c.Partitions = append(c.Partitions, m.partNames[p])
			c.States = append(c.States, st)
			c.Ops = append(c.Ops, kinds[opKind[o]])
		}
	}
	return rounds, nil
}

func (m *movesB200) free() { C.blance_moves_free(b200(), m.h) }

// ---- auditing a map (blance_map_audit; include/blance_b200.h "auditing a partition map") ------------------------
// What PlanNextMapEx never reports about a finished map: unmet constraints, copies / top copies / sole copies per
// node and NodeHierarchy name, and the failover spread.  UNTESTED GO; the C ABI underneath is covered by
// tests/test_audit_gpu.py and its C++ twin (host_api.cpp AuditMap) by tests/test_audit_host_gpu.py.
type mapAuditB200 struct {
	ShortSlots, OverSlots                  map[string]int64 // per model state
	DomTop, DomAll, DomCopies              map[string]int64 // per node or hierarchy name
	ShortParts, RuleMissParts, NoTopParts  int64
	FailoverMax                            int32
	FailoverMaxFrom, FailoverMaxTo         string
}

// auditMapB200 audits pmap against model (constraints as PlanNextMapEx would use them).  nodeHierarchy (may be nil) is
// the fault-domain forest: node ids first, then its other names in byte order; a name without a parent, or whose
// parent is "", is a root.  To have the hierarchy rules checked too, fill has_hier_rules / n_rules / n_hier_bits /
// rule_off / ie_mask of the blance_plan_in exactly as planNextMapExB200 does and read rule_miss / rule_tested.
func auditMapB200(pmap PartitionMap, nodesAll []string, model PartitionModel, nodeHierarchy map[string]string,
	failoverSpread bool) (*mapAuditB200, error) {
	var a cArena
	defer a.free()
	states := sortStateNames(model)
	S := len(states)
	it := &interner{ids: map[string]int32{}}
	for _, n := range nodesAll {
		it.get(n)
	}
	parts := partitionOrder(pmap, pmap)
	// slot ranges: max(constraints, longest list) per state
	width := make([]int, S)
	for s, st := range states {
		width[s] = model[st].Constraints
		for _, p := range pmap {
			if l := len(p.NodesByState[st]); l > width[s] {
				width[s] = l
			}
		}
		if width[s] < 0 {
			width[s] = 0
		}
	}
	cSlot, slot := a.i32(S+1, 0)
	cK, k := a.i32(S, 0)
	for s, st := range states {
		slot[s+1] = slot[s] + int32(width[s])
		k[s] = int32(model[st].Constraints)
	}
	SL := int(slot[S])
	cRows, rows := a.i32(len(parts)*SL, -1)
	cShape, shape := a.u8(len(parts) * S)
	for pi, name := range parts {
		for s, st := range states {
			l, ok := pmap[name].NodesByState[st]
			switch {
			case !ok:
				shape[pi*S+s] = C.BLANCE_SHAPE_ABSENT
			case l == nil:
				shape[pi*S+s] = C.BLANCE_SHAPE_NIL
			default:
				shape[pi*S+s] = C.BLANCE_SHAPE_LIST
			}
			for j, n := range l {
				rows[pi*SL+int(slot[s])+j] = it.get(n)
			}
		}
	}
	NU := len(it.names)
	// the forest
	vertex := append([]string(nil), it.names...)
	vid := map[string]int32{}
	for i, n := range vertex {
		vid[n] = int32(i)
	}
	var others []string
	for c, p := range nodeHierarchy {
		others = append(others, c, p)
	}
	sort.Strings(others)
	for _, n := range others {
		if _, ok := vid[n]; !ok && n != "" {
			vid[n] = int32(len(vertex))
			vertex = append(vertex, n)
		}
	}
	var opts C.blance_audit_opts
	if failoverSpread {
		opts.flags = C.BLANCE_AUDIT_N2N
	}
	if nodeHierarchy != nil {
		cPar, par := a.i32(len(vertex), -1)
		for c, p := range nodeHierarchy {
			if c != "" && p != "" {
				par[vid[c]] = vid[p]
			}
		}
		opts.n_domains = C.int32_t(len(vertex) - NU)
		opts.domain_parent = cPar
	}
	var in C.blance_plan_in
	in.n_nodes, in.n_node_ids = C.int32_t(len(nodesAll)), C.int32_t(NU)
	in.n_states, in.n_parts, in.n_slots = C.int32_t(S), C.int32_t(len(parts)), C.int32_t(SL)
	in.top_state = 0 // sortStateNames puts the top-priority state first (plan.go:126-132)
	in.state_constraints, in.state_slot_off = cK, cSlot
	V := len(vertex)
	i64 := func(n int) (*C.int64_t, []int64) {
		p := C.calloc(C.size_t(n+1), 8)
		a.ptrs = append(a.ptrs, p)
		return (*C.int64_t)(p), unsafe.Slice((*int64)(p), n+1)[:n]
	}
	var out C.blance_audit_out
	var short, over, top, all, copies []int64
	out.short_slots, short = i64(S)
	out.over_slots, over = i64(S)
	out.dom_top, top = i64(V)
	out.dom_all, all = i64(V)
	out.dom_copies, copies = i64(V)
	if st := C.blance_map_audit(b200(), &in, cRows, cShape, &opts, &out); st != C.BLANCE_OK {
		return nil, fmt.Errorf("blance_map_audit: %s", C.GoString(C.blance_last_error(b200())))
	}
	r := &mapAuditB200{ShortSlots: map[string]int64{}, OverSlots: map[string]int64{}, DomTop: map[string]int64{},
		DomAll: map[string]int64{}, DomCopies: map[string]int64{},
		ShortParts: int64(out.short_parts), RuleMissParts: int64(out.rule_miss_parts), NoTopParts: int64(out.no_top_parts)}
	for s, st := range states {
		if short[s] != 0 {
			r.ShortSlots[st] = short[s]
		}
		if over[s] != 0 {
			r.OverSlots[st] = over[s]
		}
	}
	for v, n := range vertex {
		if top[v] != 0 {
			r.DomTop[n] = top[v]
		}
		if all[v] != 0 {
			r.DomAll[n] = all[v]
		}
		if copies[v] != 0 {
			r.DomCopies[n] = copies[v]
		}
	}
	if failoverSpread && out.n2n_max_a >= 0 {
		r.FailoverMax = int32(out.n2n_max)
		r.FailoverMaxFrom, r.FailoverMaxTo = it.names[out.n2n_max_a], it.names[out.n2n_max_b]
	}
	return r, nil
}
