//go:build cgo

// Package allocategpu: the Go side of libvcalloc.so (include/vcalloc.h) for volcano's scheduler.
//
// NOT COMPILED in the build image of this repository (no Go toolchain there); written against
// volcano.sh/volcano/pkg/scheduler. It is the complete marshalling
// ("encodeSession") the Python mirror volcano_b200/snapshot.py::encode_cluster implements and the parity tests
// drive; field by field the two do the same thing, and every array below is one field of include/vcalloc.h.
//
// encode.go    framework.Session -> structure of arrays (dimension-major float64 rows, bitsets, rank keys)
// action.go    framework.Action "allocate" (+ backfill / preempt / reclaim) on top of it, incremental node rows
package allocategpu

/*
#include "vcalloc.h"
*/
import "C"

import (
	"sort"
	"strconv"
	"strings"

	v1 "k8s.io/api/core/v1"

	"volcano.sh/volcano/pkg/scheduler/api"
	"volcano.sh/volcano/pkg/scheduler/conf"
	"volcano.sh/volcano/pkg/scheduler/framework"
)

// session is the encoded framework.Session. Slices are Go memory; cgo pins them for the duration of the calls that take
// their address (vc_snapshot_upload copies everything it is handed).
type session struct {
	ssn *framework.Session

	dimNames  []v1.ResourceName // 0 cpu, 1 memory, then the scalar names sorted (api/resource_info.go:86-127 units)
	kdimNames []v1.ResourceName // cpu, memory, nvidia.com/gpu: what the upstream scorers look at
	podsDim   int

	nodes     []*api.NodeInfo // ssn.NodeList order
	tasks     []*api.TaskInfo // Pending, not BestEffort, not gated (allocate.go:255-271)
	bfTasks   []*api.TaskInfo // Pending BestEffort (backfill.go:140-151)
	runTasks  []*api.TaskInfo // node.Tasks entries in Bound / Running status (victim candidates)
	jobs      []*api.JobInfo
	jobIndex  map[api.JobID]int
	queues    []*api.QueueInfo
	queueIdx  map[api.QueueID]int
	roleOff   []int32          // [J+1]
	roleIndex []map[string]int // per job: TaskRole -> row

	dims C.vc_dims
	conf C.vc_conf

	outOfScope string // non-empty: a feature the device path does not model; the shim runs the stock action instead
	nominated  []int32 // per pending task: index of Pod.Status.NominatedNodeName in ssn.NodeList, -1 none (allocate.go:624-634)

	// vc_nodes
	nAlloc, nIdle, nUsed, nRel, nPip, nKAlloc, nKReq, nKNz []float64
	nMaxTasks, nPodCount, nZone                              []int32
	nLabels, nTaintHard, nTaintSoft                          []uint64
	nFlags                                                   []uint32
	zoneActive                                               []uint8
	// vc_tasks (pending), backfill list, running list share the layout
	t, b taskArrays
	rt   runArrays
	// vc_classes
	cSel, cAff, cTolH, cTolS, cPref []uint64
	cNAff, cNPref, cPrefW            []int32
	cFlags                           []uint32
	// vc_jobs
	jQueue, jMin, jPrio, jNTasks, jReady, jWaiting, jPBE, jValid, jTaskMinTotal []int32
	jCreation                                                                   []int64
	jUIDRank, jFlags                                                            []uint32
	jAllocated                                                                  []float64
	rMin, rOcc, rPip, rPendingOther, rValid                                     []int32
	rFlags                                                                      []uint32
	// vc_queues
	qWeight, qPrio                                  []int32
	qCreation                                       []int64
	qUIDRank, qFlags, qCapHas, qGuarHas, qReqHas, qAllocHas []uint32
	qCap, qGuar, qAlloc, qReq                       []float64
	tFlags                                          []uint32
	// vc_hdrf (drf's enableHierarchy): hdrf false = the option is off and the table is cleared
	hdrf                    bool
	hdPathOff, hdPathName   []int32
	hdNWeights              []int32
	hdWeight, hdJobRequest  []float64
}

type taskArrays struct {
	req, kreq, knz        []float64
	has, uidRank          []uint32
	job, class, role, prio []int32
	podIndex, creation    []int64
}
type runArrays struct {
	taskArrays
	node  []int32
	flags []uint32
}

// ---- helpers -------------------------------------------------------------------------------------------------------

func (e *session) dimOf(name v1.ResourceName) int {
	for i, n := range e.dimNames {
		if n == name {
			return i
		}
	}
	return -1
}

// resource vector of an api.Resource in the session's dimension order + the key set of its ScalarResources map
func (e *session) vec(r *api.Resource) ([]float64, uint32) {
	v := make([]float64, len(e.dimNames))
	var has uint32
	if r == nil {
		return v, 0
	}
	v[0], v[1] = r.MilliCPU, r.Memory
	for name, q := range r.ScalarResources {
		if d := e.dimOf(name); d >= 2 {
			v[d] = q
			has |= 1 << uint(d)
		}
	}
	return v, has
}

func putCol(dst []float64, count, idx int, v []float64) {
	for d, x := range v {
		dst[d*count+idx] = x
	}
}

// rank of every key in byte-string order (the order helpers compare UIDs in, session_plugins.go:676-682,725-731)
func ranks(keys []string) []uint32 {
	idx := make([]int, len(keys))
	for i := range idx {
		idx[i] = i
	}
	sort.SliceStable(idx, func(a, b int) bool { return keys[idx[a]] < keys[idx[b]] })
	out := make([]uint32, len(keys))
	for r, i := range idx {
		out[i] = uint32(r)
	}
	return out
}

// helpers.GetPodIndexUnderTask + strconv.Atoi (pkg/controllers/job/helpers/helpers.go:44-57); -1 = no numeric suffix
func podIndex(name string) int64 {
	parts := strings.Split(name, "-")
	if len(parts) >= 3 {
		if n, err := strconv.Atoi(parts[len(parts)-1]); err == nil && n >= 0 {
			return int64(n)
		}
	}
	return -1
}

// upstream request of a pod as noderesources computes it: Requested flavour and NonZero flavour (100m / 200Mi defaults)
func (e *session) k8sReq(pod *v1.Pod) (req, nz []float64) {
	req, nz = make([]float64, len(e.kdimNames)), make([]float64, len(e.kdimNames))
	for _, c := range pod.Spec.Containers {
		for k, name := range e.kdimNames {
			q, ok := c.Resources.Requests[name]
			var val float64
			if ok {
				if name == v1.ResourceCPU {
					val = float64(q.MilliValue())
				} else {
					val = float64(q.Value())
				}
			}
			req[k] += val
			if !ok && name == v1.ResourceCPU {
				val = 100
			}
			if !ok && name == v1.ResourceMemory {
				val = 200 * 1024 * 1024
			}
			nz[k] += val
		}
	}
	return
}

// ---- label requirements, taints and classes --------------------------------------------------------------------------

type requirement struct {
	key, op string
	values  string // sorted, comma-joined
}

type bitTable struct {
	bits map[requirement]int
	reqs []v1.NodeSelectorRequirement
}

func (bt *bitTable) bitOf(r v1.NodeSelectorRequirement) int {
	vals := append([]string(nil), r.Values...)
	sort.Strings(vals)
	k := requirement{r.Key, string(r.Operator), strings.Join(vals, ",")}
	if b, ok := bt.bits[k]; ok {
		return b
	}
	b := len(bt.reqs)
	bt.bits[k] = b
	bt.reqs = append(bt.reqs, r)
	return b
}

func setBit(words []uint64, stride, row, bit int) { words[row*stride+bit/64] |= 1 << uint(bit%64) }

// ---- encodeSession ---------------------------------------------------------------------------------------------------

func encodeSession(ssn *framework.Session, enqueueConfigured bool) *session {
	e := &session{ssn: ssn, nodes: ssn.NodeList, jobIndex: map[api.JobID]int{}, queueIdx: map[api.QueueID]int{}}

	// dimensions: cpu, memory, then every scalar name seen on a node or in a request, sorted
	scalar := map[v1.ResourceName]bool{"pods": true}
	addNames := func(r *api.Resource) {
		if r != nil {
			for n := range r.ScalarResources {
				scalar[n] = true
			}
		}
	}
	for _, n := range e.nodes {
		addNames(n.Allocatable)
	}
	for _, j := range ssn.Jobs {
		for _, t := range j.Tasks {
			addNames(t.Resreq)
		}
	}
	for _, q := range ssn.Queues {
		if q.Queue != nil {
			addNames(api.NewResource(q.Queue.Spec.Capability))
		}
	}
	names := make([]string, 0, len(scalar))
	for n := range scalar {
		names = append(names, string(n))
	}
	sort.Strings(names)
	e.dimNames = []v1.ResourceName{v1.ResourceCPU, v1.ResourceMemory}
	for _, n := range names {
		e.dimNames = append(e.dimNames, v1.ResourceName(n))
	}
	e.podsDim = e.dimOf("pods")
	e.kdimNames = []v1.ResourceName{v1.ResourceCPU, v1.ResourceMemory, "nvidia.com/gpu"}
	R, K := len(e.dimNames), len(e.kdimNames)

	// jobs and queues in a stable order (ssn.Jobs / ssn.Queues are maps; the library only needs consistent indices)
	for id := range ssn.Queues {
		e.queues = append(e.queues, ssn.Queues[id])
	}
	sort.Slice(e.queues, func(a, b int) bool { return e.queues[a].UID < e.queues[b].UID })
	for i, q := range e.queues {
		e.queueIdx[q.UID] = i
	}
	for id := range ssn.Jobs {
		e.jobs = append(e.jobs, ssn.Jobs[id])
	}
	sort.Slice(e.jobs, func(a, b int) bool { return e.jobs[a].UID < e.jobs[b].UID })
	for i, j := range e.jobs {
		e.jobIndex[j.UID] = i
	}
	J, Q, N := len(e.jobs), len(e.queues), len(e.nodes)

	// role tables + the three task lists
	e.roleOff = make([]int32, J+1)
	e.roleIndex = make([]map[string]int, J)
	type roleRow struct {
		min, occ, pip, pendingOther, valid int32
		flags                              uint32
	}
	var roles []roleRow
	for ji, job := range e.jobs {
		rows := map[string]int{}
		base := int(e.roleOff[ji])
		row := func(name string) int {
			if r, ok := rows[name]; ok {
				return r
			}
			rr := roleRow{}
			if name == "" {
				rr.flags |= C.VC_ROLE_EMPTY_NAME
			}
			if m, ok := job.TaskMinAvailable[name]; ok {
				rr.flags |= C.VC_ROLE_IN_MIN_MAP
				rr.min = m
			}
			rows[name] = base + len(rows)
			roles = append(roles, rr)
			return rows[name]
		}
		for name := range job.TaskMinAvailable {
			row(name)
		}
		for _, t := range job.Tasks {
			r := &roles[row(t.TaskRole)]
			switch {
			case api.AllocatedStatus(t.Status) || t.Status == api.Succeeded:
				r.occ++
				r.valid++
			case t.Status == api.Pipelined:
				r.pip++
				r.valid++
			case t.Status == api.Pending:
				r.valid++
				if t.BestEffort {
					r.occ++ // getJobAllocatedRoles counts pending BestEffort tasks (job_info.go:969-990)
					r.pendingOther++
				} else if t.SchGated {
					r.pendingOther++
				}
			}
			if t.Status == api.Pending && !t.SchGated {
				if t.BestEffort {
					e.bfTasks = append(e.bfTasks, t)
				} else {
					e.tasks = append(e.tasks, t)
				}
			}
		}
		e.roleIndex[ji] = rows
		e.roleOff[ji+1] = int32(base + len(rows))
	}
	for _, n := range e.nodes {
		for _, t := range n.Tasks {
			if t.Status == api.Running || t.Status == api.Bound {
				e.runTasks = append(e.runTasks, t)
			}
		}
	}
	sort.Slice(e.runTasks, func(a, b int) bool { return e.runTasks[a].UID < e.runTasks[b].UID })
	NR := len(roles)

	// label requirement / taint bit tables over everything the pending pods ask for
	lt := &bitTable{bits: map[requirement]int{}}
	hard, soft := map[v1.Taint]int{}, map[v1.Taint]int{}
	for _, n := range e.nodes {
		for _, t := range n.Node.Spec.Taints {
			key := v1.Taint{Key: t.Key, Value: t.Value, Effect: t.Effect}
			if t.Effect == v1.TaintEffectPreferNoSchedule {
				if _, ok := soft[key]; !ok {
					soft[key] = len(soft)
				}
			} else if _, ok := hard[key]; !ok {
				hard[key] = len(hard)
			}
		}
	}
	type classDef struct {
		sel      []int
		aff      [][]int
		pref     [][]int
		prefW    []int32
		tolH     []int
		tolS     []int
		unsched  bool
		revocable bool
	}
	classKey := func(c classDef) string {
		var sb strings.Builder
		w := func(xs []int) {
			for _, x := range xs {
				sb.WriteString(strconv.Itoa(x))
				sb.WriteByte(',')
			}
			sb.WriteByte(';')
		}
		w(c.sel)
		for _, t := range c.aff {
			w(t)
		}
		sb.WriteByte('|')
		for i, t := range c.pref {
			sb.WriteString(strconv.Itoa(int(c.prefW[i])))
			w(t)
		}
		w(c.tolH)
		w(c.tolS)
		sb.WriteString(strconv.FormatBool(c.unsched))
		sb.WriteString(strconv.FormatBool(c.revocable))
		return sb.String()
	}
	classOf := map[string]int{}
	var classes []classDef
	classify := func(t *api.TaskInfo) int32 {
		pod := t.Pod
		var c classDef
		for k, v := range pod.Spec.NodeSelector {
			c.sel = append(c.sel, lt.bitOf(v1.NodeSelectorRequirement{Key: k, Operator: v1.NodeSelectorOpIn, Values: []string{v}}))
		}
		sort.Ints(c.sel)
		if a := pod.Spec.Affinity; a != nil && a.NodeAffinity != nil {
			if req := a.NodeAffinity.RequiredDuringSchedulingIgnoredDuringExecution; req != nil {
				for _, term := range req.NodeSelectorTerms {
					var bits []int
					for _, r := range term.MatchExpressions {
						bits = append(bits, lt.bitOf(r))
					}
					sort.Ints(bits)
					c.aff = append(c.aff, bits)
				}
			}
			for _, p := range a.NodeAffinity.PreferredDuringSchedulingIgnoredDuringExecution {
				var bits []int
				for _, r := range p.Preference.MatchExpressions {
					bits = append(bits, lt.bitOf(r))
				}
				sort.Ints(bits)
				c.pref = append(c.pref, bits)
				c.prefW = append(c.prefW, p.Weight)
			}
		}
		for taint, bit := range hard {
			for i := range pod.Spec.Tolerations {
				if pod.Spec.Tolerations[i].ToleratesTaint(&taint) {
					c.tolH = append(c.tolH, bit)
					break
				}
			}
		}
		for taint, bit := range soft {
			for i := range pod.Spec.Tolerations {
				tol := &pod.Spec.Tolerations[i]
				if (tol.Effect == "" || tol.Effect == v1.TaintEffectPreferNoSchedule) && tol.ToleratesTaint(&taint) {
					c.tolS = append(c.tolS, bit)
					break
				}
			}
		}
		sort.Ints(c.tolH)
		sort.Ints(c.tolS)
		unsched := v1.Taint{Key: v1.TaintNodeUnschedulable, Effect: v1.TaintEffectNoSchedule}
		for i := range pod.Spec.Tolerations {
			if pod.Spec.Tolerations[i].ToleratesTaint(&unsched) {
				c.unsched = true
			}
		}
		c.revocable = len(t.RevocableZone) > 0
		k := classKey(c)
		if id, ok := classOf[k]; ok {
			return int32(id)
		}
		classOf[k] = len(classes)
		classes = append(classes, c)
		return int32(len(classes) - 1)
	}

	fill := func(list []*api.TaskInfo, a *taskArrays, withClass bool) {
		n := len(list)
		a.req, a.kreq, a.knz = make([]float64, R*n), make([]float64, K*n), make([]float64, K*n)
		a.has, a.job, a.class, a.role, a.prio = make([]uint32, n), make([]int32, n), make([]int32, n), make([]int32, n), make([]int32, n)
		a.podIndex, a.creation = make([]int64, n), make([]int64, n)
		uids := make([]string, n)
		for i, t := range list {
			v, has := e.vec(t.Resreq)
			putCol(a.req, n, i, v)
			a.has[i] = has
			kr, kn := e.k8sReq(t.Pod)
			putCol(a.kreq, n, i, kr)
			putCol(a.knz, n, i, kn)
			ji, ok := e.jobIndex[t.Job]
			if !ok {
				a.job[i], a.role[i] = -1, -1
			} else {
				a.job[i] = int32(ji)
				a.role[i] = int32(e.roleIndex[ji][t.TaskRole])
			}
			if withClass {
				a.class[i] = classify(t)
			}
			a.prio[i] = t.Priority
			a.podIndex[i] = podIndex(t.Name)
			a.creation[i] = t.Pod.CreationTimestamp.UnixNano()
			uids[i] = string(t.UID)
		}
		a.uidRank = ranks(uids)
	}
	fill(e.tasks, &e.t, true)
	fill(e.bfTasks, &e.b, true)
	fill(e.runTasks, &e.rt.taskArrays, false)
	if len(classes) == 0 {
		classes = append(classes, classDef{})
	}
	e.tFlags = make([]uint32, len(e.tasks))
	for i, t := range e.tasks {
		if p := t.Pod.Spec.PreemptionPolicy; p != nil && *p == v1.PreemptNever {
			e.tFlags[i] |= C.VC_TASK_PREEMPT_NEVER
		}
	}
	nodeIndex := map[string]int{}
	for i, n := range e.nodes {
		nodeIndex[n.Name] = i
	}
	// Pod.Status.NominatedNodeName -> index in ssn.NodeList (allocate.go:626-627: a name outside ssn.Nodes counts as none)
	for i, t := range e.tasks {
		if name := t.Pod.Status.NominatedNodeName; len(name) > 0 {
			if e.nominated == nil {
				e.nominated = make([]int32, len(e.tasks))
				for k := range e.nominated {
					e.nominated[k] = -1
				}
			}
			if ni, ok := nodeIndex[name]; ok {
				e.nominated[i] = int32(ni)
			}
		}
	}
	e.rt.node, e.rt.flags = make([]int32, len(e.runTasks)), make([]uint32, len(e.runTasks))
	for i, t := range e.runTasks {
		e.rt.node[i] = int32(nodeIndex[t.NodeName])
		if t.Status == api.Running {
			e.rt.flags[i] |= C.VC_RT_RUNNING
		} else {
			e.rt.flags[i] |= C.VC_RT_BOUND
		}
		if t.Preemptable {
			e.rt.flags[i] |= C.VC_RT_PREEMPTABLE
		}
		if t.BestEffort {
			e.rt.flags[i] |= C.VC_RT_BEST_EFFORT
		}
		cn := t.Pod.Spec.PriorityClassName
		if cn == "system-cluster-critical" || cn == "system-node-critical" || t.Namespace == "kube-system" {
			e.rt.flags[i] |= C.VC_RT_CRITICAL
		}
	}

	// classes -> bitsets
	Wl, Wt := (len(lt.reqs)+63)/64, (maxInt(len(hard), len(soft))+63)/64
	if Wl == 0 {
		Wl = 1
	}
	if Wt == 0 {
		Wt = 1
	}
	C_ := len(classes)
	MT := int(C.VC_MAX_TERMS)
	e.cSel, e.cAff, e.cPref = make([]uint64, C_*Wl), make([]uint64, C_*MT*Wl), make([]uint64, C_*MT*Wl)
	e.cTolH, e.cTolS = make([]uint64, C_*Wt), make([]uint64, C_*Wt)
	e.cNAff, e.cNPref, e.cPrefW, e.cFlags = make([]int32, C_), make([]int32, C_), make([]int32, C_*MT), make([]uint32, C_)
	for ci, c := range classes {
		for _, b := range c.sel {
			setBit(e.cSel, Wl, ci, b)
		}
		e.cNAff[ci] = int32(len(c.aff))
		for k, term := range c.aff {
			for _, b := range term {
				setBit(e.cAff, Wl, ci*MT+k, b)
			}
		}
		e.cNPref[ci] = int32(len(c.pref))
		for k, term := range c.pref {
			for _, b := range term {
				setBit(e.cPref, Wl, ci*MT+k, b)
			}
			e.cPrefW[ci*MT+k] = c.prefW[k]
		}
		for _, b := range c.tolH {
			setBit(e.cTolH, Wt, ci, b)
		}
		for _, b := range c.tolS {
			setBit(e.cTolS, Wt, ci, b)
		}
		if c.revocable {
			e.cFlags[ci] |= C.VC_CLASS_REVOCABLE
		}
		if c.unsched {
			e.cFlags[ci] |= C.VC_CLASS_TOLERATES_UNSCHEDULABLE
		}
	}

	// nodes
	e.nAlloc, e.nIdle, e.nUsed, e.nRel, e.nPip = make([]float64, R*N), make([]float64, R*N), make([]float64, R*N), make([]float64, R*N), make([]float64, R*N)
	e.nKAlloc, e.nKReq, e.nKNz = make([]float64, K*N), make([]float64, K*N), make([]float64, K*N)
	e.nMaxTasks, e.nPodCount, e.nZone, e.nFlags = make([]int32, N), make([]int32, N), make([]int32, N), make([]uint32, N)
	e.nLabels, e.nTaintHard, e.nTaintSoft = make([]uint64, Wl*N), make([]uint64, Wt*N), make([]uint64, Wt*N)
	zones := map[string]int{}
	for i, n := range e.nodes {
		e.encodeNodeRows(i, n)
		e.nMaxTasks[i] = int32(n.Allocatable.MaxTaskNum)
		lbls := nodeLabels(n.Node.Labels)
		for b, r := range lt.reqs {
			if matches(lbls, r) {
				e.nLabels[(b/64)*N+i] |= 1 << uint(b%64)
			}
		}
		for _, t := range n.Node.Spec.Taints {
			key := v1.Taint{Key: t.Key, Value: t.Value, Effect: t.Effect}
			if t.Effect == v1.TaintEffectPreferNoSchedule {
				b := soft[key]
				e.nTaintSoft[(b/64)*N+i] |= 1 << uint(b%64)
			} else {
				b := hard[key]
				e.nTaintHard[(b/64)*N+i] |= 1 << uint(b%64)
			}
		}
		if n.Node.Spec.Unschedulable {
			e.nFlags[i] |= C.VC_NODE_UNSCHEDULABLE
		}
		e.nZone[i] = -1
		if n.RevocableZone != "" {
			z, ok := zones[n.RevocableZone]
			if !ok {
				z = len(zones)
				zones[n.RevocableZone] = z
			}
			e.nZone[i] = int32(z)
		}
	}
	e.zoneActive = make([]uint8, maxInt(len(zones), 1))
	for z, zi := range zones {
		if tdmZoneActive(ssn, z) { // tdm.availableRevocableZone(z) == nil, evaluated once per cycle (tdm.go:118-137)
			e.zoneActive[zi] = 1
		}
	}

	// jobs
	e.jQueue, e.jMin, e.jPrio, e.jNTasks = make([]int32, J), make([]int32, J), make([]int32, J), make([]int32, J)
	e.jReady, e.jWaiting, e.jPBE, e.jValid, e.jTaskMinTotal = make([]int32, J), make([]int32, J), make([]int32, J), make([]int32, J), make([]int32, J)
	e.jCreation, e.jFlags, e.jAllocated = make([]int64, J), make([]uint32, J), make([]float64, R*J)
	jobKeys := make([]string, J)
	for ji, job := range e.jobs {
		q, ok := e.queueIdx[job.Queue]
		if !ok {
			q = -1
		}
		e.jQueue[ji], e.jMin[ji], e.jPrio[ji] = int32(q), job.MinAvailable, job.Priority
		e.jNTasks[ji] = int32(len(job.Tasks))
		e.jReady[ji], e.jWaiting[ji] = job.ReadyTaskNum(), job.WaitingTaskNum()
		e.jPBE[ji], e.jValid[ji] = job.PendingBestEffortTaskNum(), job.ValidTaskNum()
		e.jTaskMinTotal[ji] = job.TaskMinAvailableTotal
		e.jCreation[ji] = job.CreationTimestamp.UnixNano()
		jobKeys[ji] = string(job.UID)
		if job.IsPending() {
			e.jFlags[ji] |= C.VC_JOB_PENDING_PHASE
		}
		if job.Preemptable {
			e.jFlags[ji] |= C.VC_JOB_PREEMPTABLE
		}
		if job.ContainsHardTopology() || job.ContainsSubJobPolicy() {
			e.jFlags[ji] |= C.VC_JOB_UNSUPPORTED
		}
		alloc := api.EmptyResource() // drf attr.allocated: AllocatedStatus tasks (drf.go:196-203)
		for _, t := range job.Tasks {
			if api.AllocatedStatus(t.Status) {
				alloc.Add(t.Resreq)
			}
		}
		v, _ := e.vec(alloc)
		putCol(e.jAllocated, J, ji, v)
	}
	e.jUIDRank = ranks(jobKeys)
	e.rMin, e.rOcc, e.rPip, e.rPendingOther, e.rValid, e.rFlags = make([]int32, NR), make([]int32, NR), make([]int32, NR), make([]int32, NR), make([]int32, NR), make([]uint32, NR)
	for i, r := range roles {
		e.rMin[i], e.rOcc[i], e.rPip[i], e.rPendingOther[i], e.rValid[i], e.rFlags[i] = r.min, r.occ, r.pip, r.pendingOther, r.valid, r.flags
	}

	// queues: spec + proportion's allocated / request sums (proportion.go:143-156)
	e.qWeight, e.qPrio, e.qCreation, e.qFlags = make([]int32, Q), make([]int32, Q), make([]int64, Q), make([]uint32, Q)
	e.qCap, e.qGuar, e.qAlloc, e.qReq = make([]float64, R*Q), make([]float64, R*Q), make([]float64, R*Q), make([]float64, R*Q)
	e.qCapHas, e.qGuarHas, e.qReqHas, e.qAllocHas = make([]uint32, Q), make([]uint32, Q), make([]uint32, Q), make([]uint32, Q)
	queueKeys := make([]string, Q)
	for qi, q := range e.queues {
		e.qWeight[qi] = q.Weight
		queueKeys[qi] = string(q.UID)
		if q.Queue != nil {
			e.qPrio[qi] = q.Queue.Spec.Priority
			e.qCreation[qi] = q.Queue.CreationTimestamp.UnixNano()
			if q.Queue.Status.State == "Open" {
				e.qFlags[qi] |= C.VC_QUEUE_OPEN
			}
			if !q.Reclaimable() {
				e.qFlags[qi] |= C.VC_QUEUE_NOT_RECLAIMABLE
			}
			if len(q.Queue.Spec.Capability) != 0 {
				v, has := e.vec(api.NewResource(q.Queue.Spec.Capability))
				putCol(e.qCap, Q, qi, v)
				e.qCapHas[qi] = has | C.VC_RES_HAS_ANY
			}
			if len(q.Queue.Spec.Guarantee.Resource) != 0 {
				v, has := e.vec(api.NewResource(q.Queue.Spec.Guarantee.Resource))
				putCol(e.qGuar, Q, qi, v)
				e.qGuarHas[qi] = has | C.VC_RES_HAS_ANY
			}
		}
	}
	e.qUIDRank = ranks(queueKeys)
	for _, job := range e.jobs {
		qi, ok := e.queueIdx[job.Queue]
		if !ok {
			continue
		}
		for _, t := range job.Tasks {
			v, has := e.vec(t.Resreq)
			if api.AllocatedStatus(t.Status) {
				for d := range v {
					e.qAlloc[d*Q+qi] += v[d]
					e.qReq[d*Q+qi] += v[d]
				}
				e.qAllocHas[qi] |= has
				e.qReqHas[qi] |= has
			} else if t.Status == api.Pending {
				for d := range v {
					e.qReq[d*Q+qi] += v[d]
				}
				e.qReqHas[qi] |= has
			}
		}
	}

	e.dims = C.vc_dims{n_nodes: C.int32_t(N), n_tasks: C.int32_t(len(e.tasks)), n_jobs: C.int32_t(J), n_queues: C.int32_t(Q),
		n_classes: C.int32_t(C_), n_roles: C.int32_t(NR), n_dims: C.int32_t(R), n_kdims: C.int32_t(K),
		label_words: C.int32_t(Wl), taint_words: C.int32_t(Wt), n_zones: C.int32_t(len(zones)), pods_dim: C.int32_t(e.podsDim)}
	e.encodeConf(ssn.Tiers, enqueueConfigured)
	if e.hdrf {
		e.encodeHdrf(R)
	}
	return e
}

// encodeHdrf fills vc_hdrf: per queue the segments of QueueInfo.Hierarchy below the root as interned names, the number of
// weight segments below the root and strconv.ParseFloat of each (the value it returns even with an error: the library
// clamps it as buildHierarchy does, drf.go:458-500); per job JobInfo.TotalRequest. Tree construction and the refusal of
// what the reference crashes on are the library's.
func (e *session) encodeHdrf(R int) {
	Q, J := len(e.queues), len(e.jobs)
	names := map[string]int32{}
	e.hdPathOff = make([]int32, Q+1)
	e.hdNWeights = make([]int32, Q)
	e.hdPathName, e.hdWeight = nil, nil
	for qi, q := range e.queues {
		paths := strings.Split(q.Hierarchy, "/")[1:]
		weights := strings.Split(q.Weights, "/")[1:]
		for i, seg := range paths {
			id, ok := names[seg]
			if !ok {
				id = int32(len(names))
				names[seg] = id
			}
			e.hdPathName = append(e.hdPathName, id)
			w := 0.0
			if i < len(weights) {
				w, _ = strconv.ParseFloat(weights[i], 64)
			}
			e.hdWeight = append(e.hdWeight, w)
		}
		e.hdNWeights[qi] = int32(len(weights))
		e.hdPathOff[qi+1] = int32(len(e.hdPathName))
	}
	e.hdJobRequest = make([]float64, R*J)
	for ji, job := range e.jobs {
		v, _ := e.vec(job.TotalRequest)
		putCol(e.hdJobRequest, J, ji, v)
	}
}

// the accounting rows of one node: the part vc_snapshot_update_nodes re-uploads when NodeInfo.Generation moved
func (e *session) encodeNodeRows(i int, n *api.NodeInfo) {
	N, R := len(e.nodes), len(e.dimNames)
	for _, p := range []struct {
		dst []float64
		r   *api.Resource
	}{{e.nAlloc, n.Allocatable}, {e.nIdle, n.Idle}, {e.nUsed, n.Used}, {e.nRel, n.Releasing}, {e.nPip, n.Pipelined}} {
		v, _ := e.vec(p.r)
		for d := 0; d < R; d++ {
			p.dst[d*N+i] = v[d]
		}
	}
	if ki, ok := e.ssn.NodeMap[n.Name]; ok { // the k8s NodeInfo the upstream scorers read (framework/util.go:226-234)
		al, rq, nz := ki.GetAllocatable(), ki.GetRequested(), ki.GetNonZeroRequested()
		e.nKAlloc[0*N+i], e.nKAlloc[1*N+i] = float64(al.GetMilliCPU()), float64(al.GetMemory())
		e.nKReq[0*N+i], e.nKReq[1*N+i] = float64(rq.GetMilliCPU()), float64(rq.GetMemory())
		e.nKNz[0*N+i], e.nKNz[1*N+i] = float64(nz.GetMilliCPU()), float64(nz.GetMemory())
		for k := 2; k < len(e.kdimNames); k++ {
			e.nKAlloc[k*N+i] = float64(al.GetScalarResources()[e.kdimNames[k]])
			e.nKReq[k*N+i] = float64(rq.GetScalarResources()[e.kdimNames[k]])
		}
		e.nPodCount[i] = int32(len(ki.GetPods()))
	}
}

// conf.Tiers -> vc_conf: plugin order, Enabled* flags (after ApplyPluginConfDefaults, plugins/defaults.go:29-55), arguments
func (e *session) encodeConf(tiers []conf.Tier, enqueueConfigured bool) {
	c := &e.conf
	ids := map[string]C.int32_t{"priority": C.VC_PLUGIN_PRIORITY, "gang": C.VC_PLUGIN_GANG, "drf": C.VC_PLUGIN_DRF,
		"proportion": C.VC_PLUGIN_PROPORTION, "predicates": C.VC_PLUGIN_PREDICATES, "nodeorder": C.VC_PLUGIN_NODEORDER,
		"binpack": C.VC_PLUGIN_BINPACK, "tdm": C.VC_PLUGIN_TDM, "network-topology-aware": C.VC_PLUGIN_NETWORK_TOPOLOGY_AWARE,
		"conformance": C.VC_PLUGIN_CONFORMANCE, "pdb": C.VC_PLUGIN_PDB, "cdp": C.VC_PLUGIN_CDP}
	on := func(b *bool) bool { return b != nil && *b }
	c.binpack_weight = 1
	for d := range c.binpack_dim_weight {
		c.binpack_dim_weight[d], c.nta_dim_weight[d] = -1, -1
	}
	c.w_least, c.w_most, c.w_balanced, c.w_node_affinity, c.w_taint_toleration = 1, 0, 1, 2, 3
	c.predicates_enable = C.VC_PRED_NODE_AFFINITY | C.VC_PRED_TAINT_TOLERATION
	c.nta_weight, c.nta_normal_pod_enable, c.nta_fading = 1, 1, 0.8
	n := 0
	for ti, tier := range tiers {
		for _, p := range tier.Plugins {
			if n >= int(C.VC_MAX_PLUGINS) {
				break
			}
			id, ok := ids[p.Name]
			if !ok {
				id = C.VC_PLUGIN_OTHER
			}
			if p.Name == "drf" && on(p.EnabledHierarchy) { // hdrf: queue order from the hierarchy tree (drf/drf.go:147-156)
				e.hdrf = true
			}
			var en C.uint32_t
			for flag, b := range map[C.uint32_t]*bool{C.VC_EN_JOB_ORDER: p.EnabledJobOrder, C.VC_EN_JOB_READY: p.EnabledJobReady,
				C.VC_EN_JOB_PIPELINED: p.EnabledJobPipelined, C.VC_EN_TASK_ORDER: p.EnabledTaskOrder,
				C.VC_EN_QUEUE_ORDER: p.EnabledQueueOrder, C.VC_EN_PREDICATE: p.EnabledPredicate, C.VC_EN_NODE_ORDER: p.EnabledNodeOrder,
				C.VC_EN_BEST_NODE: p.EnabledBestNode, C.VC_EN_OVERUSED: p.EnabledOverused, C.VC_EN_ALLOCATABLE: p.EnabledAllocatable,
				C.VC_EN_PREEMPTABLE: p.EnabledPreemptable, C.VC_EN_RECLAIMABLE: p.EnabledReclaimable,
				C.VC_EN_JOB_STARVING: p.EnabledJobStarving, C.VC_EN_PREEMPTIVE: p.EnablePreemptive} {
				if on(b) {
					en |= flag
				}
			}
			c.plugins[n] = C.vc_plugin_option{plugin: id, tier: C.int32_t(ti), enabled: en}
			n++
			e.encodeArguments(p.Name, framework.Arguments(p.Arguments))
		}
	}
	c.n_plugins = C.int32_t(n)
	for k, name := range e.kdimNames {
		c.kdim_dim[k] = C.int32_t(e.dimOf(name))
	}
	c.enable_predicate_error_cache = 1
	if enqueueConfigured {
		c.enqueue_action_enabled = 1
	}
	c.percentage_nodes_to_find, c.min_nodes_to_find, c.min_percentage_nodes_to_find = serverOptions()
	c.last_processed_node_index = C.int32_t(lastProcessedNodeIndex) // carried from the previous cycle (action.go)
}

func (e *session) encodeArguments(plugin string, a framework.Arguments) {
	c := &e.conf
	geti := func(key string, def int) C.int32_t { v := def; a.GetInt(&v, key); return C.int32_t(v) }
	nonneg := func(v C.int32_t) C.int32_t {
		if v < 0 {
			return 1
		}
		return v
	}
	weights := func(prefix, list string, cpuKey, memKey string) map[string]C.int32_t {
		w := map[string]C.int32_t{"cpu": nonneg(geti(cpuKey, 1)), "memory": nonneg(geti(memKey, 1))}
		if s, ok := a[list].(string); ok {
			for _, r := range strings.Split(s, ",") {
				if r = strings.TrimSpace(r); r != "" {
					w[r] = nonneg(geti(prefix+r, 1))
				}
			}
		}
		return w
	}
	switch plugin {
	case "binpack": // plugins/binpack/binpack.go:94-158
		c.binpack_weight = geti("binpack.weight", 1)
		w := weights("binpack.resources.", "binpack.resources", "binpack.cpu", "binpack.memory")
		for d, name := range e.dimNames {
			if x, ok := w[string(name)]; ok {
				c.binpack_dim_weight[d] = x
			}
		}
	case "nodeorder": // plugins/nodeorder/nodeorder.go:131-171
		c.w_node_affinity, c.w_least = geti("nodeaffinity.weight", 2), geti("leastrequested.weight", 1)
		c.w_most, c.w_balanced = geti("mostrequested.weight", 0), geti("balancedresource.weight", 1)
		c.w_taint_toleration = geti("tainttoleration.weight", 3)
	case "predicates": // plugins/predicates/predicates.go:126-151
		na, tt := true, true
		a.GetBool(&na, "predicate.NodeAffinityEnable")
		a.GetBool(&tt, "predicate.TaintTolerationEnable")
		c.predicates_enable = 0
		if na {
			c.predicates_enable |= C.VC_PRED_NODE_AFFINITY
		}
		if tt {
			c.predicates_enable |= C.VC_PRED_TAINT_TOLERATION
		}
	case "network-topology-aware": // network_topology_aware.go:155-229
		c.nta_weight = nonneg(geti("weight", 1))
		w := weights("hypernode.binpack.resources.", "hypernode.binpack.resources", "hypernode.binpack.cpu", "hypernode.binpack.memory")
		for d, name := range e.dimNames {
			if x, ok := w[string(name)]; ok {
				c.nta_dim_weight[d] = x
			}
		}
		en, fading := true, 0.8
		a.GetBool(&en, "hypernode.binpack.normal-pod.enable")
		a.GetFloat64(&fading, "hypernode.binpack.normal-pod.fading")
		if fading < 0 {
			fading = 0.8
		}
		if !en {
			c.nta_normal_pod_enable = 0
		}
		c.nta_fading = C.double(fading)
	}
}

func maxInt(a, b int) int {
	if a > b {
		return a
	}
	return b
}
