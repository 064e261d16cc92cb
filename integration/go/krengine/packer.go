package krengine

/*
#include "kr_engine.h"
*/
import "C"

import (
	"fmt"
	"unsafe"
)

// PodObj is what the path reads of a *corev1.Pod (kr_pod_obj): the caller evaluates the few predicates that need the typed object
// (shouldDeletePod's container-status lookup, FindHeadPodReadyCondition) and passes plain values.
type PodObj struct {
	Namespace, Name                          string
	Cluster, Group                           string // labels ray.io/cluster, ray.io/group
	ReplicaName, ReplicaIndex                string // labels ray.io/worker-group-replica-name / -index (text; parsed like strconv.Atoi inside)
	NodeType, Phase, ReadyCond               uint8  // KR_NT_*, KR_PHASE_*, KR_COND_* (absent condition: KR_COND_ABSENT)
	RestartNever, RayTerminated, HasDeletion bool
	HeadReadyStatus                          uint8  // the rest only for head Pods: utils.FindHeadPodReadyCondition
	HeadReadyReason, HeadReadyMessage        string
	PodIP, RecreateHash, KubeRayVersion      string // status.podIP; annotations ray.io/upgrade-strategy-recreate-hash, ray.io/kuberay-version
	HasRecreateHash, HasKubeRayVersion       bool   // the annotation is present (an empty value is not the same as none)
}

// GroupObj is one WorkerGroupSpec as the path reads it.
type GroupObj struct {
	Name                                         string
	Replicas, MinReplicas, MaxReplicas, NumHosts int32
	Flags                                        uint32 // KR_GF_*: replicas nil, suspend, expectation satisfied, ...
	WorkersToDelete                              []string
}

// ClusterObj is a RayCluster as the path reads it: identity and epoch keys, the old status calculateStatus compares against, the head
// Service the controller found, the worker groups and the spec as JSON (muted and canonicalised inside, once per generation).
type ClusterObj struct {
	Namespace, Name, UID        string
	ResourceVersion, Generation uint64
	Flags                       uint32 // KR_CF_*
	SuspendStatus, ExtErrKind   uint8
	OldState, SvcCount, SvcIPKind uint8
	ExtErrMessage               string
	OldCounts                   [5]int32
	OldCondStatus, OldCondVariant [5]uint8
	OldHeadReadyReason, OldHeadReadyMessage, OldReplicaFailureMessage string
	OldHead                     [4]string // podIP, serviceIP, podName, serviceName
	SvcIP, SvcName, StatusSummary string
	Groups                      []GroupObj
	SpecJSON                    []byte // json.Marshal(instance.Spec)
}

// Packer is the native event-driven packer (kr_packer_*): informer handlers upsert / delete objects as events arrive, Flush uploads what
// moved since the last epoch, Engine() runs the pass.  One goroutine at a time.
type Packer struct {
	h   *C.kr_packer
	eng *Engine
}

func NewPacker(capacities Config, kubeRayVersion string) (*Packer, error) {
	cc := capacities.c()
	var h *C.kr_packer
	if rc := C.kr_packer_create(&cc, &h); rc != C.KR_OK {
		return nil, fmt.Errorf("krengine: kr_packer_create failed (%d)", int(rc))
	}
	p := &Packer{h: h, eng: &Engine{h: C.kr_packer_engine(h)}}
	var s strs
	defer s.release()
	if rc := C.kr_packer_set_kuberay_version(h, s.str(kubeRayVersion)); rc != C.KR_OK {
		p.Close()
		return nil, p.err(rc)
	}
	return p, nil
}

func (p *Packer) Close()          { C.kr_packer_destroy(p.h); p.h = nil }
func (p *Packer) Engine() *Engine { return p.eng }
func (p *Packer) err(rc C.int) error {
	return fmt.Errorf("krengine: packer: %s (%d)", C.GoString(C.kr_packer_last_error(p.h)), int(rc))
}

func (p *Packer) UpsertPod(o *PodObj) error {
	var s strs
	defer s.release()
	c := o.c(&s)
	if rc := C.kr_packer_pod_upsert(p.h, &c); rc != C.KR_OK {
		return p.err(rc)
	}
	return nil
}

// c fills the kr_pod_obj; its strings stay pinned until s.release().
func (o *PodObj) c(s *strs) C.kr_pod_obj {
	c := C.kr_pod_obj{ns: s.str(o.Namespace), name: s.str(o.Name), cluster: s.str(o.Cluster), group: s.str(o.Group), replica_name: s.str(o.ReplicaName),
		replica_index: s.str(o.ReplicaIndex), node_type: C.uint8_t(o.NodeType), phase: C.uint8_t(o.Phase), ready_cond: C.uint8_t(o.ReadyCond),
		restart_never: b2u(o.RestartNever), ray_terminated: b2u(o.RayTerminated), has_deletion_ts: b2u(o.HasDeletion), head_ready_status: C.uint8_t(o.HeadReadyStatus),
		head_ready_reason: s.str(o.HeadReadyReason), head_ready_msg: s.str(o.HeadReadyMessage), pod_ip: s.str(o.PodIP)}
	if o.HasRecreateHash {
		c.recreate_hash = s.present(o.RecreateHash)
	}
	if o.HasKubeRayVersion {
		c.kuberay_version = s.present(o.KubeRayVersion)
	}
	return c
}

func (p *Packer) DeletePod(ns, name string) error {
	var s strs
	defer s.release()
	if rc := C.kr_packer_pod_delete(p.h, s.str(ns), s.str(name)); rc != C.KR_OK {
		return p.err(rc)
	}
	return nil
}

func (p *Packer) UpsertCluster(o *ClusterObj) error {
	var s strs
	defer s.release()
	c := o.c(&s)
	if rc := C.kr_packer_cluster_upsert(p.h, &c); rc != C.KR_OK {
		return p.err(rc)
	}
	return nil
}

// c fills the kr_cluster_obj; its strings, groups, name lists and spec stay pinned until s.release().
func (o *ClusterObj) c(s *strs) C.kr_cluster_obj {
	groups := make([]C.kr_group_obj, len(o.Groups))
	names := make([][]C.kr_str, len(o.Groups)) // one C-visible array of names per group, pinned below
	for i := range o.Groups {
		g := &o.Groups[i]
		groups[i] = C.kr_group_obj{name: s.str(g.Name), replicas: C.int32_t(g.Replicas), min_replicas: C.int32_t(g.MinReplicas), max_replicas: C.int32_t(g.MaxReplicas),
			num_hosts: C.int32_t(g.NumHosts), flags: C.uint32_t(g.Flags), n_workers_to_delete: C.uint32_t(len(g.WorkersToDelete))}
		if len(g.WorkersToDelete) > 0 {
			names[i] = make([]C.kr_str, len(g.WorkersToDelete))
			for k, w := range g.WorkersToDelete {
				names[i][k] = s.str(w)
			}
			s.pin.Pin(&names[i][0])
			groups[i].workers_to_delete = &names[i][0]
		}
	}
	c := C.kr_cluster_obj{ns: s.str(o.Namespace), name: s.str(o.Name), uid: s.str(o.UID), resource_version: C.uint64_t(o.ResourceVersion), generation: C.uint64_t(o.Generation),
		flags: C.uint32_t(o.Flags), suspend_status: C.uint8_t(o.SuspendStatus), ext_err_kind: C.uint8_t(o.ExtErrKind), old_state: C.uint8_t(o.OldState),
		svc_count: C.uint8_t(o.SvcCount), svc_ip_kind: C.uint8_t(o.SvcIPKind), ext_err_msg: s.str(o.ExtErrMessage),
		old_head_ready_reason: s.str(o.OldHeadReadyReason), old_head_ready_msg: s.str(o.OldHeadReadyMessage), old_replica_failure_msg: s.str(o.OldReplicaFailureMessage),
		svc_ip: s.str(o.SvcIP), svc_name: s.str(o.SvcName), status_summary: s.str(o.StatusSummary), n_groups: C.uint32_t(len(groups))}
	for k := 0; k < 5; k++ {
		c.old_counts[k] = C.int32_t(o.OldCounts[k])
		c.old_cond_status[k] = C.uint8_t(o.OldCondStatus[k])
		c.old_cond_variant[k] = C.uint8_t(o.OldCondVariant[k])
	}
	for k := 0; k < 4; k++ {
		c.old_head[k] = s.str(o.OldHead[k])
	}
	if len(groups) > 0 {
		s.pin.Pin(&groups[0])
		c.groups = &groups[0]
	}
	if len(o.SpecJSON) > 0 {
		s.pin.Pin(&o.SpecJSON[0])
		c.spec_json = (*C.uint8_t)(unsafe.Pointer(&o.SpecJSON[0]))
		c.spec_json_len = C.uint64_t(len(o.SpecJSON))
	}
	return c
}

func (p *Packer) DeleteCluster(ns, name string) error {
	var s strs
	defer s.release()
	if rc := C.kr_packer_cluster_delete(p.h, s.str(ns), s.str(name)); rc != C.KR_OK {
		return p.err(rc)
	}
	return nil
}

// UpsertJob / DeleteJob: the RayJob roll-up rows (rayjob_controller.go:203-216, 880-905).
func (p *Packer) UpsertJob(ns, name, clusterName, statusSummary string) error {
	var s strs
	defer s.release()
	j := C.kr_job_obj{ns: s.str(ns), name: s.str(name), cluster_name: s.str(clusterName), status_summary: s.str(statusSummary)}
	if rc := C.kr_packer_job_upsert(p.h, &j); rc != C.KR_OK {
		return p.err(rc)
	}
	return nil
}

func (p *Packer) DeleteJob(ns, name string) error {
	var s strs
	defer s.release()
	if rc := C.kr_packer_job_delete(p.h, s.str(ns), s.str(name)); rc != C.KR_OK {
		return p.err(rc)
	}
	return nil
}

// PackSpecRows is the Flush mode bit of a flush that committed re-emitted specs row by row (OptSpecRows) instead of KR_PART_JSON.
const PackSpecRows = uint32(C.KR_PACK_SPEC_ROWS)

// PackJsonMoves is the Flush mode bit of a flush that committed a compaction of its JSON arena as moves inside the device arena
// (OptJsonMoves) instead of KR_PART_JSON.
const PackJsonMoves = uint32(C.KR_PACK_JSON_MOVES)

// Flush uploads what moved since the last flush; mode reports how (KR_PACK_FULL | KR_PACK_POD_ROWS | KR_PACK_OBJECT_ROWS |
// KR_PACK_SPEC_ROWS | KR_PACK_JSON_MOVES | KR_PART_*).
func (p *Packer) Flush() (mode uint32, err error) {
	var m C.uint32_t
	if rc := C.kr_packer_flush(p.h, &m); rc != C.KR_OK {
		return 0, p.err(rc)
	}
	var sz C.kr_sizes
	if rc := C.kr_packer_sizes(p.h, &sz); rc != C.KR_OK {
		return 0, p.err(rc)
	}
	p.eng.sizes = Sizes{Clusters: uint32(sz.n_clusters), Groups: uint32(sz.n_groups), Wtd: uint32(sz.n_wtd), Pods: uint32(sz.n_pods), Heads: uint32(sz.n_heads),
		Jobs: uint32(sz.n_jobs), JSONBytes: uint64(sz.json_bytes)}
	return uint32(m), nil
}

// Intern returns the id of a string (the two HeadPodReady texts of Flags); String turns an id in a record back into text.
func (p *Packer) Intern(v string) uint32 {
	var s strs
	defer s.release()
	return uint32(C.kr_packer_intern(p.h, s.present(v)))
}

func (p *Packer) String(id uint32) string {
	var out C.kr_str
	if C.kr_packer_string(p.h, C.uint32_t(id), &out) != C.KR_OK || out.p == nil {
		return ""
	}
	return C.GoStringN(out.p, C.int(out.n))
}

// ClusterRow / PodKey translate between objects and arena rows: -1 when the RayCluster is not packed; act_pod_idx -> the Pod to delete.
func (p *Packer) ClusterRow(ns, name string) int64 {
	var s strs
	defer s.release()
	return int64(C.kr_packer_cluster_row(p.h, s.str(ns), s.str(name)))
}

func (p *Packer) PodKey(row uint32) (ns, name string, ok bool) {
	var a, b C.kr_str
	if C.kr_packer_pod_key(p.h, C.uint32_t(row), &a, &b) != C.KR_OK {
		return "", "", false
	}
	return C.GoStringN(a.p, C.int(a.n)), C.GoStringN(b.p, C.int(b.n)), true
}

// Epoch keys (SURVEY §8(b)): Reconcile(req) trusts the record of req only if its own cache read of the RayCluster shows the
// resourceVersion packed here and no Pod event arrived since the flush.
func (p *Packer) Epoch() (epoch, podsetVersion uint64) {
	var e, v C.uint64_t
	C.kr_packer_epoch(p.h, &e, &v)
	return uint64(e), uint64(v)
}

func (p *Packer) ClusterEpoch(row uint32) (resourceVersion, generation uint64) {
	var rv, g C.uint64_t
	C.kr_packer_cluster_epoch(p.h, C.uint32_t(row), &rv, &g)
	return uint64(rv), uint64(g)
}
