//go:build cgo

package allocategpu

/*
#cgo CFLAGS: -I${SRCDIR}/../../../include
#cgo LDFLAGS: -L${SRCDIR}/../../../volcano_b200 -lvcalloc
#include "vcalloc.h"
#include <stdlib.h>
*/
import "C"

import (
	"math"
	"math/rand"
	"strconv"
	"time"
	"unsafe"

	v1 "k8s.io/api/core/v1"
	policyv1 "k8s.io/api/policy/v1"
	metav1 "k8s.io/apimachinery/pkg/apis/meta/v1"
	"k8s.io/apimachinery/pkg/labels"
	"k8s.io/klog/v2"

	"volcano.sh/apis/pkg/apis/scheduling/v1beta1"
	"volcano.sh/volcano/cmd/scheduler/app/options"
	stockallocate "volcano.sh/volcano/pkg/scheduler/actions/allocate"
	stockbackfill "volcano.sh/volcano/pkg/scheduler/actions/backfill"
	stockpreempt "volcano.sh/volcano/pkg/scheduler/actions/preempt"
	stockreclaim "volcano.sh/volcano/pkg/scheduler/actions/reclaim"
	"volcano.sh/volcano/pkg/scheduler/api"
	"volcano.sh/volcano/pkg/scheduler/conf"
	"volcano.sh/volcano/pkg/scheduler/framework"
)

// util.lastProcessedNodeIndex of the reference is a package variable (util/scheduler_helper.go:50); the library returns
// the value a cycle leaves in vc_stats and takes it back through vc_conf.
var lastProcessedNodeIndex int32

func serverOptions() (C.int32_t, C.int32_t, C.int32_t) {
	o := options.ServerOpts
	return C.int32_t(o.PercentageOfNodesToFind), C.int32_t(o.MinNodesToFind), C.int32_t(o.MinPercentageOfNodesToFind)
}

func nodeLabels(l map[string]string) map[string]string { return l }

// v1.NodeSelectorRequirement against node labels (nodeaffinity helper semantics: In, NotIn, Exists, DoesNotExist, Gt, Lt)
func matches(labels map[string]string, r v1.NodeSelectorRequirement) bool {
	val, ok := labels[r.Key]
	switch r.Operator {
	case v1.NodeSelectorOpIn:
		for _, x := range r.Values {
			if ok && x == val {
				return true
			}
		}
		return false
	case v1.NodeSelectorOpNotIn:
		for _, x := range r.Values {
			if ok && x == val {
				return false
			}
		}
		return true
	case v1.NodeSelectorOpExists:
		return ok
	case v1.NodeSelectorOpDoesNotExist:
		return !ok
	case v1.NodeSelectorOpGt, v1.NodeSelectorOpLt:
		if !ok || len(r.Values) != 1 {
			return false
		}
		a, e1 := strconv.ParseInt(val, 10, 64)
		b, e2 := strconv.ParseInt(r.Values[0], 10, 64)
		if e1 != nil || e2 != nil {
			return false
		}
		if r.Operator == v1.NodeSelectorOpGt {
			return a > b
		}
		return a < b
	}
	return false
}

// tdm.availableRevocableZone(zone) == nil as of now (plugins/tdm/tdm.go:118-137); the shim asks the configured tdm plugin
func tdmZoneActive(ssn *framework.Session, zone string) bool { return tdmZoneAvailable(ssn, zone) }

// ---------------------------------------------------------------------------------------------------------------------

// cycle is the device-side session the actions of one scheduling cycle share (all run on the cycle goroutine,
// scheduler.go:124-153). It survives across cycles: when the pending set is unchanged only the node rows whose
// NodeInfo.Generation moved are uploaded (vc_snapshot_update_nodes).
type cycle struct {
	snap      *C.vc_snapshot
	enc       *session
	nodeGen   map[string]int64 // NodeInfo.Generation as uploaded
	taskSig   string           // identity of the uploaded pending set + jobs + queues + conf
	allocated bool
}

var cur cycle

func enqueueConfigured() bool { return conf.EnabledActionMap["enqueue"] }

func signature(e *session) string {
	h := uint64(1469598103934665603)
	mix := func(s string) {
		for i := 0; i < len(s); i++ {
			h ^= uint64(s[i])
			h *= 1099511628211
		}
	}
	for _, t := range e.tasks {
		mix(string(t.UID))
		mix(t.Pod.Status.NominatedNodeName) // a new nomination is a new session for the device
	}
	for _, j := range e.jobs {
		mix(string(j.UID))
		mix(strconv.Itoa(int(j.ReadyTaskNum())))
	}
	for _, q := range e.queues {
		mix(string(q.UID))
	}
	return strconv.FormatUint(h, 16) + ":" + strconv.Itoa(len(e.nodes))
}

func ptrF(s []float64) *C.double {
	if len(s) == 0 {
		return nil
	}
	return (*C.double)(unsafe.Pointer(&s[0]))
}
func ptrI(s []int32) *C.int32_t {
	if len(s) == 0 {
		return nil
	}
	return (*C.int32_t)(unsafe.Pointer(&s[0]))
}
func ptrL(s []int64) *C.int64_t {
	if len(s) == 0 {
		return nil
	}
	return (*C.int64_t)(unsafe.Pointer(&s[0]))
}
func ptrU(s []uint32) *C.uint32_t {
	if len(s) == 0 {
		return nil
	}
	return (*C.uint32_t)(unsafe.Pointer(&s[0]))
}
func ptrQ(s []uint64) *C.uint64_t {
	if len(s) == 0 {
		return nil
	}
	return (*C.uint64_t)(unsafe.Pointer(&s[0]))
}
func ptrB(s []uint8) *C.uint8_t {
	if len(s) == 0 {
		return nil
	}
	return (*C.uint8_t)(unsafe.Pointer(&s[0]))
}

func (e *session) cNodes() C.vc_nodes {
	return C.vc_nodes{allocatable: ptrF(e.nAlloc), idle: ptrF(e.nIdle), used: ptrF(e.nUsed), releasing: ptrF(e.nRel),
		pipelined: ptrF(e.nPip), k8s_allocatable: ptrF(e.nKAlloc), k8s_requested: ptrF(e.nKReq), k8s_nonzero_requested: ptrF(e.nKNz),
		max_tasks: ptrI(e.nMaxTasks), pod_count: ptrI(e.nPodCount), label_bits: ptrQ(e.nLabels), taint_hard: ptrQ(e.nTaintHard),
		taint_soft: ptrQ(e.nTaintSoft), flags: ptrU(e.nFlags), revocable_zone: ptrI(e.nZone), zone_active: ptrB(e.zoneActive)}
}
func (a *taskArrays) c() C.vc_tasks {
	return C.vc_tasks{resreq: ptrF(a.req), req_has: ptrU(a.has), k8s_req: ptrF(a.kreq), k8s_nonzero_req: ptrF(a.knz), job: ptrI(a.job),
		klass: ptrI(a.class), role: ptrI(a.role), priority: ptrI(a.prio), pod_index: ptrL(a.podIndex), creation_ts: ptrL(a.creation),
		uid_rank: ptrU(a.uidRank)}
}
func (e *session) cClasses() C.vc_classes {
	return C.vc_classes{selector: ptrQ(e.cSel), n_affinity: ptrI(e.cNAff), affinity: ptrQ(e.cAff), tolerated_hard: ptrQ(e.cTolH),
		tolerated_soft: ptrQ(e.cTolS), n_preferred: ptrI(e.cNPref), preferred: ptrQ(e.cPref), preferred_weight: ptrI(e.cPrefW),
		flags: ptrU(e.cFlags)}
}
func (e *session) cJobs() C.vc_jobs {
	return C.vc_jobs{queue: ptrI(e.jQueue), min_available: ptrI(e.jMin), priority: ptrI(e.jPrio), creation_ts: ptrL(e.jCreation),
		uid_rank: ptrU(e.jUIDRank), flags: ptrU(e.jFlags), n_tasks_total: ptrI(e.jNTasks), ready_num: ptrI(e.jReady),
		waiting_num: ptrI(e.jWaiting), pending_besteffort: ptrI(e.jPBE), valid_num: ptrI(e.jValid), task_min_total: ptrI(e.jTaskMinTotal),
		role_off: ptrI(e.roleOff), allocated: ptrF(e.jAllocated), role_min: ptrI(e.rMin), role_occupied: ptrI(e.rOcc),
		role_pipelined: ptrI(e.rPip), role_pending_other: ptrI(e.rPendingOther), role_valid: ptrI(e.rValid), role_flags: ptrU(e.rFlags)}
}
func (e *session) cQueues() C.vc_queues {
	return C.vc_queues{weight: ptrI(e.qWeight), priority: ptrI(e.qPrio), creation_ts: ptrL(e.qCreation), uid_rank: ptrU(e.qUIDRank),
		flags: ptrU(e.qFlags), capability: ptrF(e.qCap), capability_has: ptrU(e.qCapHas), guarantee: ptrF(e.qGuar),
		guarantee_has: ptrU(e.qGuarHas), allocated: ptrF(e.qAlloc), request: ptrF(e.qReq), request_has: ptrU(e.qReqHas),
		allocated_has: ptrU(e.qAllocHas)}
}
func (e *session) cRunning() C.vc_running_tasks {
	a := &e.rt
	return C.vc_running_tasks{n_tasks: C.int32_t(len(e.runTasks)), node: ptrI(a.node), job: ptrI(a.job), role: ptrI(a.role),
		priority: ptrI(a.prio), pod_index: ptrL(a.podIndex), creation_ts: ptrL(a.creation), uid_rank: ptrU(a.uidRank),
		resreq: ptrF(a.req), req_has: ptrU(a.has), k8s_req: ptrF(a.kreq), k8s_nonzero_req: ptrF(a.knz), flags: ptrU(a.flags)}
}

func fail(what string) { klog.Errorf("vcalloc %s: %s", what, C.GoString(C.vc_last_error())) }

// openCycle: encode the session and bring the device session up to date — a full upload, or the dirty node rows only
func openCycle(ssn *framework.Session) bool {
	e := encodeSession(ssn, enqueueConfigured())
	if e.outOfScope != "" {
		klog.V(3).Infof("vcalloc: %s is outside the device path, the stock action runs this cycle", e.outOfScope)
		return false
	}
	sig := signature(e)
	if cur.snap != nil && cur.taskSig == sig && cur.enc != nil && cur.enc.dims == e.dims {
		// same pending set, jobs, queues: upload the rows of the nodes whose Generation moved (api/node_info.go:95-99)
		var idx []int32
		for i, n := range e.nodes {
			if cur.nodeGen[n.Name] != n.Generation {
				idx = append(idx, int32(i))
			}
		}
		m, R, K, N := len(idx), len(e.dimNames), len(e.kdimNames), len(e.nodes)
		gather := func(src []float64, rows int) []float64 {
			out := make([]float64, rows*m)
			for d := 0; d < rows; d++ {
				for k, i := range idx {
					out[d*m+k] = src[d*N+int(i)]
				}
			}
			return out
		}
		idle, used, rel, pip := gather(e.nIdle, R), gather(e.nUsed, R), gather(e.nRel, R), gather(e.nPip, R)
		kreq, knz := gather(e.nKReq, K), gather(e.nKNz, K)
		pods := make([]int32, m)
		for k, i := range idx {
			pods[k] = e.nPodCount[i]
		}
		rows := C.vc_nodes{idle: ptrF(idle), used: ptrF(used), releasing: ptrF(rel), pipelined: ptrF(pip), k8s_requested: ptrF(kreq),
			k8s_nonzero_requested: ptrF(knz), pod_count: ptrI(pods)}
		if rc := C.vc_snapshot_update_nodes(cur.snap, C.int32_t(m), ptrI(idx), &rows); rc == 0 {
			for _, n := range e.nodes {
				cur.nodeGen[n.Name] = n.Generation
			}
			cur.enc, cur.allocated = e, false
			return true
		} // VC_EUNSUPPORTED (topology tables, first Releasing resource): fall through to the full upload
	}
	if cur.snap != nil && (cur.enc == nil || cur.enc.dims != e.dims) {
		C.vc_snapshot_destroy(cur.snap)
		cur.snap = nil
	}
	if cur.snap == nil {
		if rc := C.vc_snapshot_create(&e.dims, &cur.snap); rc != 0 {
			fail("create")
			return false
		}
	}
	if topo := e.hypernodes(); topo != nil {
		if rc := C.vc_snapshot_set_topology(cur.snap, topo); rc != 0 {
			fail("topology")
			return false
		}
	}
	var hd *C.vc_hdrf // nil clears the table
	if e.hdrf {
		hd = &C.vc_hdrf{path_off: ptrI(e.hdPathOff), path_name: ptrI(e.hdPathName), n_weights: ptrI(e.hdNWeights),
			weight: ptrF(e.hdWeight), job_request: ptrF(e.hdJobRequest)}
	}
	if rc := C.vc_snapshot_set_hdrf(cur.snap, hd); rc != 0 {
		fail("hdrf table")
		return false
	}
	bf := e.b.c()
	if rc := C.vc_snapshot_set_backfill(cur.snap, C.int32_t(len(e.bfTasks)), &bf); rc != 0 {
		fail("backfill list")
		return false
	}
	rt := e.cRunning()
	if rc := C.vc_snapshot_set_running(cur.snap, &rt, ptrU(e.tFlags)); rc != 0 {
		fail("running tasks")
		return false
	}
	if rc := C.vc_snapshot_set_nominated(cur.snap, ptrI(e.nominated)); rc != 0 { // nil clears the list
		fail("nominated nodes")
		return false
	}
	nd, tk, cl, jb, qu := e.cNodes(), e.t.c(), e.cClasses(), e.cJobs(), e.cQueues()
	if rc := C.vc_snapshot_upload(cur.snap, &nd, &tk, &cl, &jb, &qu, &e.conf); rc != 0 {
		fail("upload")
		return false
	}
	cur.enc, cur.taskSig, cur.allocated = e, sig, false
	cur.nodeGen = make(map[string]int64, len(e.nodes))
	for _, n := range e.nodes {
		cur.nodeGen[n.Name] = n.Generation
	}
	return true
}

// ---- the allocate action ---------------------------------------------------------------------------------------------

type Action struct{}

func New() *Action             { return &Action{} }
func (a *Action) Name() string { return "allocate" }
func (a *Action) Initialize() {
	if C.vc_abi_version() != C.VC_ABI_VERSION {
		panic("libvcalloc.so does not match the vcalloc.h this shim was compiled against")
	}
	if rc := C.vc_init(0); rc != 0 {
		panic(C.GoString(C.vc_last_error())) // no CUDA device: the library has no CPU path
	}
}
func (a *Action) UnInitialize() {}

// runStock: the session is outside the device path (hdrf, an upload the library refused, ...): the reference's own action
// runs this cycle, and so do the follow-up actions of the same session (the device session does not see what it did)
var stockSession *framework.Session

func runStock(name string, ssn *framework.Session) {
	stockSession = ssn
	var act framework.Action
	switch name {
	case "allocate":
		act = stockallocate.New()
	case "backfill":
		act = stockbackfill.New()
	case "preempt":
		act = stockpreempt.New()
	default:
		act = stockreclaim.New()
	}
	act.Initialize()
	act.Execute(ssn)
	act.UnInitialize()
}

func (a *Action) Execute(ssn *framework.Session) {
	if !openCycle(ssn) {
		runStock("allocate", ssn) // the session is untouched by the device path at this point
		return
	}
	e := cur.enc
	// buildAllocateContext rewrites Pending PodGroups to Inqueue when no enqueue action is configured (allocate.go:154-164);
	// the library assumes it (vc_backfill_run / vc_preempt_run after vc_allocate_run), the session must see it too
	if !enqueueConfigured() {
		for _, job := range e.jobs {
			if job.IsPending() {
				job.PodGroup.Status.Phase = "Inqueue"
			}
		}
	}
	var res *C.vc_result
	if rc := C.vc_allocate_run(cur.snap, &res); rc != 0 {
		fail("allocate") // e.g. VC_EUNSUPPORTED for hard-mode topology jobs: nothing was applied
		runStock("allocate", ssn)
		return
	}
	defer C.vc_result_free(res)
	cur.allocated = true
	lastProcessedNodeIndex = int32(C.vc_result_stats(res).last_processed_node_index)
	visits := unsafe.Slice(C.vc_result_visits(res), int(C.vc_result_num_visits(res)))
	decs := unsafe.Slice(C.vc_result_decisions(res), int(C.vc_result_num_decisions(res)))
	for _, v := range visits {
		if v.outcome == C.VC_VISIT_DISCARD {
			continue
		}
		stmt := framework.NewStatement(ssn)
		for _, d := range decs[v.first_op : v.first_op+v.n_ops] {
			task, node := e.tasks[d.task], e.nodes[d.node]
			if d.kind == C.VC_OP_ALLOCATE {
				if err := stmt.Allocate(task, node); err != nil { // framework/statement.go:242-302
					klog.Errorf("replay Allocate %s -> %s: %v", task.Name, node.Name, err)
				}
			} else if err := stmt.Pipeline(task, node.Name, false); err != nil { // framework/statement.go:146-200
				klog.Errorf("replay Pipeline %s -> %s: %v", task.Name, node.Name, err)
			}
		}
		if v.outcome == C.VC_VISIT_COMMIT {
			stmt.Commit() // statement.go:384-412 -> cache.AddBindTask
		} // VC_VISIT_KEEP: a pipelined job keeps its operations in the session, uncommitted (allocate.go:330-331)
	}
	var nj C.size_t
	if ah := C.vc_result_job_allocated_hypernodes(res, &nj); ah != nil { // allocate.go:681-686
		for j, h := range unsafe.Slice(ah, int(nj)) {
			e.setAllocatedHyperNode(j, int(h))
		}
	}
	for _, t := range unsafe.Slice(C.vc_result_fit_errors(res), int(C.vc_result_num_fit_errors(res))) {
		e.recordFitError(int(t)) // job.NodesFitErrors[task.UID] (allocate.go:600-607, :651)
	}
}

// job.NodesFitErrors entry for a task no node took: every node with the generic "does not fit" error; the per-node
// reasons of the reference come from its predicate closures and are diagnostics only
func (e *session) recordFitError(t int) {
	task := e.tasks[t]
	job := e.ssn.Jobs[task.Job]
	if job == nil {
		return
	}
	fe := api.NewFitErrors()
	for _, n := range e.nodes {
		fe.SetNodeError(n.Name, api.NewFitError(task, n, "node(s) did not fit the task on the device path"))
	}
	job.NodesFitErrors[task.UID] = fe
}

// setPreemptOptions hands the preempt action's arguments (preempt.go:90-99) to the library, with what its topology-aware
// reading reads per running task: PodPriority (Spec.Priority, 0 when nil), Status.StartTime, one time.Now() per run and a
// seed for the offsets that rand.Intn would draw.
func setPreemptOptions(ssn *framework.Session, e *session) bool {
	args := framework.GetArgOfActionFromConf(ssn.Configurations, "preempt")
	topo, workers, pct, minAbs, maxAbs := false, 16, 10, 1, 100
	args.GetBool(&topo, stockpreempt.EnableTopologyAwarePreemptionKey)
	args.GetInt(&workers, stockpreempt.TopologyAwarePreemptWorkerNumKey) // accepted and ignored: the dry runs run at once
	args.GetInt(&pct, stockpreempt.MinCandidateNodesPercentageKey)
	args.GetInt(&minAbs, stockpreempt.MinCandidateNodesAbsoluteKey)
	args.GetInt(&maxAbs, stockpreempt.MaxCandidateNodesAbsoluteKey)
	n := len(e.runTasks)
	prio, start := make([]int32, n), make([]int64, n)
	for i, t := range e.runTasks {
		prio[i] = stockpreempt.PodPriority(t.Pod)
		start[i] = math.MinInt64 // VC_START_TIME_UNSET
		if t.Pod.Status.StartTime != nil {
			start[i] = t.Pod.Status.StartTime.UnixNano()
		}
	}
	opts := C.vc_preempt_options{topology_aware: 0, min_candidate_nodes_percentage: C.int32_t(pct),
		min_candidate_nodes_absolute: C.int32_t(minAbs), max_candidate_nodes_absolute: C.int32_t(maxAbs),
		offset_seed: C.uint64_t(rand.Uint64()), now_ns: C.int64_t(time.Now().UnixNano()), n_running: C.int32_t(n),
		rt_pod_priority: ptrI(prio), rt_start_ns: ptrL(start)}
	if topo {
		opts.topology_aware = 1
	}
	if rc := C.vc_snapshot_set_preempt_options(cur.snap, &opts); rc != 0 {
		fail("preempt options")
		return false
	}
	return true
}

// guardsVote: pdb or cdp registers a victim function the action calls (EnabledPreemptable for preempt, EnabledReclaimable
// for reclaim), the library's test for requiring the table. Other sessions skip the PDB list and the per-pod work.
func guardsVote(ssn *framework.Session, action string) bool {
	for _, tier := range ssn.Tiers {
		for _, p := range tier.Plugins {
			if p.Name != "pdb" && p.Name != "cdp" {
				continue
			}
			en := p.EnabledPreemptable
			if action == "reclaim" {
				en = p.EnabledReclaimable
			} else if action != "preempt" {
				continue
			}
			if en != nil && *en {
				return true
			}
		}
	}
	return false
}

// cooldownUntil is LastTransitionTime + cooldown in ns, saturated to the int64 range (UnixNano is undefined outside it; a
// protection end past it stays after any now, one before it is never after now)
func cooldownUntil(t time.Time) int64 {
	if t.After(time.Unix(0, math.MaxInt64)) {
		return math.MaxInt64
	}
	if t.Before(time.Unix(0, math.MinInt64+1)) {
		return math.MinInt64 // VC_COOLDOWN_NONE
	}
	return t.UnixNano()
}

// setVictimGuards hands the library what the pdb and cdp victim votes read (vc_victim_guards): the PDBs listed through the
// informer factory as getPodDisruptionBudgets does (pdb.go:143-153), matched per running pod with LabelSelectorAsSelector,
// and per pod the end of cdp's cooldown (cdp.go:56-96). One time.Now() for the session.
func setVictimGuards(ssn *framework.Session, e *session) bool {
	n := len(e.runTasks)
	var pdbs []*policyv1.PodDisruptionBudget
	if f := ssn.InformerFactory(); f != nil {
		list, err := f.Policy().V1().PodDisruptionBudgets().Lister().List(labels.Everything())
		if err != nil {
			fail("victim guards: pdb list")
			return false
		}
		pdbs = list
	}
	allowed := make([]int32, len(pdbs)+1)
	sel := make([]labels.Selector, len(pdbs))
	for i, b := range pdbs {
		allowed[i] = b.Status.DisruptionsAllowed
		if s, err := metav1.LabelSelectorAsSelector(b.Spec.Selector); err == nil && !s.Empty() {
			sel[i] = s
		}
	}
	off, list := make([]int32, n+1), make([]int32, 0, n+1)
	flags, until := make([]uint32, n+1), make([]int64, n+1)
	for i, t := range e.runTasks {
		pod := t.Pod
		if len(pod.Labels) == 0 {
			flags[i] |= C.VC_GUARD_NO_LABELS
		} else {
			for k, b := range pdbs {
				if b.Namespace != pod.Namespace || sel[k] == nil || !sel[k].Matches(labels.Set(pod.Labels)) {
					continue
				}
				if _, ok := b.Status.DisruptedPods[pod.Name]; ok {
					continue
				}
				list = append(list, int32(k))
			}
		}
		off[i+1] = int32(len(list))
		until[i] = math.MinInt64 // VC_COOLDOWN_NONE
		v, ok := pod.Labels[v1beta1.CooldownTime]
		if !ok {
			v, ok = pod.Annotations[v1beta1.CooldownTime]
		}
		if d, err := time.ParseDuration(v); ok && err == nil && pod.Status.Phase == v1.PodRunning {
			for _, c := range pod.Status.Conditions {
				if c.Type == v1.PodScheduled && c.Status == v1.ConditionTrue {
					until[i] = cooldownUntil(c.LastTransitionTime.Add(d))
					break
				}
			}
		}
	}
	list = append(list, 0) // keep the slice's pointer valid when empty
	g := C.vc_victim_guards{n_running: C.int32_t(n), n_pdb: C.int32_t(len(pdbs)), pdb_allowed: ptrI(allowed),
		rt_pdb_off: ptrI(off), rt_pdb: ptrI(list), rt_flags: ptrU(flags), rt_cooldown_until_ns: ptrL(until),
		now_ns: C.int64_t(time.Now().UnixNano())}
	if rc := C.vc_snapshot_set_victim_guards(cur.snap, &g); rc != 0 {
		fail("victim guards")
		return false
	}
	return true
}

// ---- backfill / preempt / reclaim on the same device session ------------------------------------------------------------

type followUp struct{ name string }

func NewBackfill() *followUp             { return &followUp{"backfill"} }
func NewPreempt() *followUp              { return &followUp{"preempt"} }
func NewReclaim() *followUp              { return &followUp{"reclaim"} }
func (a *followUp) Name() string         { return a.name }
func (a *followUp) Initialize()          {}
func (a *followUp) UnInitialize()        {}
func (a *followUp) Execute(ssn *framework.Session) {
	if stockSession == ssn { // an earlier action of this cycle ran on the stock path
		runStock(a.name, ssn)
		return
	}
	if cur.snap == nil || cur.enc == nil || cur.enc.ssn != ssn {
		if !openCycle(ssn) { // the action runs without allocate before it in the configured list
			runStock(a.name, ssn)
			return
		}
	}
	e := cur.enc
	var res *C.vc_result
	var rc C.int
	if guardsVote(ssn, a.name) && !setVictimGuards(ssn, e) {
		runStock(a.name, ssn)
		return
	}
	switch a.name {
	case "backfill":
		rc = C.vc_backfill_run(cur.snap, &res)
	case "preempt":
		if !setPreemptOptions(ssn, e) {
			runStock(a.name, ssn)
			return
		}
		rc = C.vc_preempt_run(cur.snap, &res)
	default:
		rc = C.vc_reclaim_run(cur.snap, &res)
	}
	if rc != 0 {
		fail(a.name) // VC_EUNSUPPORTED (tdm, BestEffort preemptors, ...): the configuration is outside the path and nothing
		// was applied (network-topology-aware sessions and soft-mode topology jobs run on the library); the session state is
		// what the earlier replays left, so the reference's action can take over from here
		runStock(a.name, ssn)
		return
	}
	defer C.vc_result_free(res)
	if a.name != "backfill" { // every PredicateNodes call of preempt / reclaim moves the index under sampling
		lastProcessedNodeIndex = int32(C.vc_result_stats(res).last_processed_node_index)
	}
	visits := unsafe.Slice(C.vc_result_visits(res), int(C.vc_result_num_visits(res)))
	decs := unsafe.Slice(C.vc_result_decisions(res), int(C.vc_result_num_decisions(res)))
	if a.name == "backfill" {
		for _, d := range decs { // decision.task indexes the list given to vc_snapshot_set_backfill
			if err := ssn.Allocate(e.bfTasks[d.task], e.nodes[d.node]); err != nil { // backfill.go:107-112
				klog.Errorf("replay backfill: %v", err)
			}
		}
		return
	}
	for _, v := range visits { // one Statement per visit (preempt.go:177-243, :246-280; reclaim.go:121-163)
		if v.outcome != C.VC_VISIT_COMMIT {
			continue
		}
		stmt := framework.NewStatement(ssn)
		evicted := false
		for _, d := range decs[v.first_op : v.first_op+v.n_ops] {
			if d.kind == C.VC_OP_EVICT {
				stmt.Evict(e.runTasks[d.task], a.name) // framework/statement.go:72-99
				evicted = true
			} else {
				if err := stmt.Pipeline(e.tasks[d.task], e.nodes[d.node].Name, evicted); err != nil {
					klog.Errorf("replay %s pipeline: %v", a.name, err)
				}
				evicted = false
			}
		}
		stmt.Commit()
	}
}
