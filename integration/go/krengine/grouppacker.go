package krengine

/*
#include "kr_engine.h"
*/
import "C"

import (
	"errors"
	"fmt"
	"unsafe"
)

// ShardOfKey is the group packer's routing rule (kr_shard_of_key): FNV-1a 64 over namespace + "/" + RayCluster name, modulo n.
// A RayCluster is routed by its own name, a Pod by its ray.io/cluster label, a RayJob by its cluster name.
func ShardOfKey(ns, clusterName string, n uint32) uint32 {
	var s strs
	defer s.release()
	return uint32(C.kr_shard_of_key(s.present(ns), s.present(clusterName), C.uint32_t(n)))
}

// GroupPacker is the native packer sharded over GPUs (kr_group_packer_*): one Packer per shard behind one handle.  The informer
// handlers call the Upsert / Delete methods as events arrive (routed natively by (namespace, RayCluster name), on the calling
// goroutine); Flush and Reconcile run every shard on its own NUMA-bound worker thread.  Shard(i) is shard i's Packer for reads
// (String, PodKey, ClusterRow, Epoch, Intern) and per-shard options (Shard(i).Engine().SetOption: they are not forwarded); the
// group packer owns the shards: Close it, never a Shard.
// One goroutine at a time.
type GroupPacker struct {
	h      *C.kr_group_packer
	shards []*Packer // views: owned by the group packer
}

// NewGroupPacker creates one packer per entry of devices (a CUDA ordinal may repeat: several shards on one GPU).
func NewGroupPacker(perShard Config, devices []int32, kubeRayVersion string) (*GroupPacker, error) {
	if len(devices) == 0 {
		return nil, errors.New("krengine: NewGroupPacker needs at least one device")
	}
	cc := perShard.c()
	var h *C.kr_group_packer
	if rc := C.kr_group_packer_create(&cc, (*C.int32_t)(unsafe.Pointer(&devices[0])), C.uint32_t(len(devices)), &h); rc != C.KR_OK {
		return nil, fmt.Errorf("krengine: kr_group_packer_create failed (%d)", int(rc))
	}
	g := &GroupPacker{h: h}
	var s strs
	defer s.release()
	for i := range devices {
		ph := C.kr_group_packer_shard(h, C.uint32_t(i))
		g.shards = append(g.shards, &Packer{h: ph, eng: &Engine{h: C.kr_packer_engine(ph)}})
		if rc := C.kr_packer_set_kuberay_version(ph, s.str(kubeRayVersion)); rc != C.KR_OK {
			err := g.shards[i].err(rc)
			g.Close()
			return nil, err
		}
	}
	return g, nil
}

// Close frees every shard (its packer and engine); the Shard views are invalid afterwards.
func (g *GroupPacker) Close() {
	C.kr_group_packer_destroy(g.h)
	g.h = nil
	for _, p := range g.shards {
		p.h, p.eng.h = nil, nil
	}
}

func (g *GroupPacker) Size() int            { return len(g.shards) }
func (g *GroupPacker) Shard(i int) *Packer { return g.shards[i] }

// ShardOf names the shard of a routing key (ShardOfKey with this group packer's size).
func (g *GroupPacker) ShardOf(ns, clusterName string) int {
	return int(ShardOfKey(ns, clusterName, uint32(len(g.shards))))
}

func (g *GroupPacker) err(rc C.int) error {
	return fmt.Errorf("krengine: group packer: %s (%d)", C.GoString(C.kr_group_packer_last_error(g.h)), int(rc))
}

func (g *GroupPacker) UpsertPod(o *PodObj) error {
	var s strs
	defer s.release()
	c := o.c(&s)
	if rc := C.kr_group_packer_pod_upsert(g.h, &c); rc != C.KR_OK {
		return g.err(rc)
	}
	return nil
}

func (g *GroupPacker) DeletePod(ns, name string) error {
	var s strs
	defer s.release()
	if rc := C.kr_group_packer_pod_delete(g.h, s.str(ns), s.str(name)); rc != C.KR_OK {
		return g.err(rc)
	}
	return nil
}

func (g *GroupPacker) UpsertCluster(o *ClusterObj) error {
	var s strs
	defer s.release()
	c := o.c(&s)
	if rc := C.kr_group_packer_cluster_upsert(g.h, &c); rc != C.KR_OK {
		return g.err(rc)
	}
	return nil
}

func (g *GroupPacker) DeleteCluster(ns, name string) error {
	var s strs
	defer s.release()
	if rc := C.kr_group_packer_cluster_delete(g.h, s.str(ns), s.str(name)); rc != C.KR_OK {
		return g.err(rc)
	}
	return nil
}

func (g *GroupPacker) UpsertJob(ns, name, clusterName, statusSummary string) error {
	var s strs
	defer s.release()
	j := C.kr_job_obj{ns: s.str(ns), name: s.str(name), cluster_name: s.str(clusterName), status_summary: s.str(statusSummary)}
	if rc := C.kr_group_packer_job_upsert(g.h, &j); rc != C.KR_OK {
		return g.err(rc)
	}
	return nil
}

func (g *GroupPacker) DeleteJob(ns, name string) error {
	var s strs
	defer s.release()
	if rc := C.kr_group_packer_job_delete(g.h, s.str(ns), s.str(name)); rc != C.KR_OK {
		return g.err(rc)
	}
	return nil
}

// Flush brings every shard's device copy up to date, in parallel; modes[i] is shard i's Packer.Flush mode.
func (g *GroupPacker) Flush() (modes []uint32, err error) {
	m := make([]C.uint32_t, len(g.shards))
	if rc := C.kr_group_packer_flush(g.h, &m[0]); rc != C.KR_OK {
		return nil, g.err(rc)
	}
	modes = make([]uint32, len(m))
	for i, p := range g.shards {
		var sz C.kr_sizes
		if rc := C.kr_packer_sizes(p.h, &sz); rc != C.KR_OK {
			return nil, p.err(rc)
		}
		p.eng.sizes = Sizes{Clusters: uint32(sz.n_clusters), Groups: uint32(sz.n_groups), Wtd: uint32(sz.n_wtd), Pods: uint32(sz.n_pods), Heads: uint32(sz.n_heads),
			Jobs: uint32(sz.n_jobs), JSONBytes: uint64(sz.json_bytes)}
		modes[i] = uint32(m[i])
	}
	return modes, nil
}

// Reconcile runs every shard's pass in parallel.  flags[i] is shard i's (HeadNotFoundReason / HeadNotFoundMessage from
// Shard(i).Intern); results[i] are shard i's records, its rows named through Shard(i).
func (g *GroupPacker) Reconcile(flags []Flags) ([]*Results, error) {
	if len(flags) != len(g.shards) {
		return nil, errors.New("krengine: GroupPacker.Reconcile wants one Flags per shard")
	}
	cf := make([]C.kr_flags, len(flags))
	for i, f := range flags {
		cf[i] = f.c()
	}
	views := make([]C.kr_results_view, len(g.shards))
	if rc := C.kr_group_packer_reconcile(g.h, &cf[0], &views[0]); rc != C.KR_OK {
		return nil, g.err(rc) // every shard's previous results are invalid now: the caller runs the per-object Go path for this epoch
	}
	out := make([]*Results, len(g.shards))
	for i, p := range g.shards {
		out[i] = wrapResults(&views[i], p.eng.sizes)
	}
	return out, nil
}
