package krengine

/*
#include "kr_engine.h"
*/
import "C"

import (
	"context"
	"sync"
	"time"
)

// Record is what Reconcile(req) receives for its RayCluster: the engine's decisions for that cluster and the epoch they belong to.
type Record struct {
	Row             uint32
	Cluster         C.kr_cluster_result
	Groups          []C.kr_group_result // the cluster's worker groups, spec order
	Hash            string              // 32 characters: the spec hash createHeadPod stamps on the head
	Deletes         []PodAction         // in the order the reference issues the Delete calls
	CreateIdx       [][]int32           // per group: replica indices to create (multi-host: one per replica group)
	ResourceVersion uint64              // the RayCluster resourceVersion the snapshot held
	PodsetVersion   uint64              // bumped by every Pod event: a newer value means the record is stale
}

// PodAction: delete this Pod for this reason (KR_ACT_*).
type PodAction struct {
	Namespace, Name string
	Code            uint8
}

type lookup struct {
	ns, name string
	reply    chan *Record
}

// Batcher owns the packer and the engine.  Informer handlers send closures that upsert / delete objects; Reconcile(req) asks for the
// record of its RayCluster.  Every Period (or as soon as a lookup finds events pending) it flushes and runs one pass; between passes
// lookups are answered from the last results when their epoch still holds.
type Batcher struct {
	Period time.Duration
	Flags  Flags

	p       *Packer
	events  chan func(*Packer)
	lookups chan lookup
	res     *Results
	podset  uint64
	mu      sync.Mutex // guards stats: a metrics scraper reads them from its own goroutine
	stats   Stats
}

// Stats counts the passes of the batcher's epochs by kind, and the full passes by cause (KR_FULL_* bit -> passes that reported
// it; one pass may report several).  What an operator's metrics code exports: a fleet whose epochs keep falling back to full passes
// shows which rule sends them there (DESIGN §4.3), and so which option or cap would keep them incremental.
type Stats struct {
	Incremental, Full uint64
	Causes            map[uint32]uint64
}

func NewBatcher(p *Packer, flags Flags, period time.Duration) *Batcher {
	return &Batcher{Period: period, Flags: flags, p: p, events: make(chan func(*Packer), 4096), lookups: make(chan lookup, 256)}
}

// Event queues an informer event (Add / Update / Delete of a Pod, RayCluster or RayJob): f runs on the batching goroutine.
func (b *Batcher) Event(f func(*Packer)) { b.events <- f }

// Lookup returns the record of (ns, name), or nil when the engine has nothing trustworthy for it: the caller then runs the original
// per-object Go path (level-triggered reconcile makes either answer safe).
func (b *Batcher) Lookup(ctx context.Context, ns, name string) *Record {
	l := lookup{ns: ns, name: name, reply: make(chan *Record, 1)}
	select {
	case b.lookups <- l:
	case <-ctx.Done():
		return nil
	}
	select {
	case r := <-l.reply:
		return r
	case <-ctx.Done():
		return nil
	}
}

// Run is the batching goroutine.
func (b *Batcher) Run(ctx context.Context) {
	tick := time.NewTicker(b.Period)
	defer tick.Stop()
	dirty := true
	for {
		select {
		case <-ctx.Done():
			return
		case f := <-b.events:
			f(b.p)
			dirty = true
		case <-tick.C:
			if dirty {
				dirty = !b.epoch()
			}
		case l := <-b.lookups:
			if dirty { // never answer from results older than an event we already hold
				dirty = !b.epoch()
			}
			l.reply <- b.record(l.ns, l.name)
		}
	}
}

// epoch: drain what is queued, flush, run one pass.  false = the pass failed; the results are dropped and lookups return nil.
func (b *Batcher) epoch() bool {
	for drained := false; !drained; {
		select {
		case f := <-b.events:
			f(b.p)
		default:
			drained = true
		}
	}
	b.res = nil
	if _, err := b.p.Flush(); err != nil {
		return false
	}
	res, err := b.p.Engine().Reconcile(b.Flags)
	if err != nil {
		return false
	}
	b.res = res
	_, b.podset = b.p.Epoch()
	if rep, err := b.p.Engine().LastPass(); err == nil {
		b.count(rep)
	}
	return true
}

func (b *Batcher) count(rep PassReport) {
	b.mu.Lock()
	defer b.mu.Unlock()
	if rep.Incremental {
		b.stats.Incremental++
		return
	}
	b.stats.Full++
	if b.stats.Causes == nil {
		b.stats.Causes = map[uint32]uint64{}
	}
	for _, c := range FullCauses {
		if rep.WhyFull&c.Bit != 0 {
			b.stats.Causes[c.Bit]++
		}
	}
}

// Stats returns a copy of the pass counters; safe from any goroutine.
func (b *Batcher) Stats() Stats {
	b.mu.Lock()
	defer b.mu.Unlock()
	s := Stats{Incremental: b.stats.Incremental, Full: b.stats.Full, Causes: map[uint32]uint64{}}
	for k, v := range b.stats.Causes {
		s.Causes[k] = v
	}
	return s
}

func (b *Batcher) record(ns, name string) *Record {
	if b.res == nil {
		return nil
	}
	row := b.p.ClusterRow(ns, name)
	if row < 0 {
		return nil
	}
	c := uint32(row)
	res := b.res
	cr := res.Clusters[c]
	rec := &Record{Row: c, Cluster: cr, Hash: string(res.Hash[32*c : 32*c+32]), PodsetVersion: b.podset}
	rec.ResourceVersion, _ = b.p.ClusterEpoch(c)
	// the compact action list: cluster c owns [act_start[c], act_start[c]+act_cnt[c]), already in the reference's call order
	start, cnt := res.ActStart[c], res.ActCnt[c]
	for i := start; i < start+cnt; i++ {
		if ns, name, ok := b.p.PodKey(res.ActPodIdx[i]); ok {
			rec.Deletes = append(rec.Deletes, PodAction{Namespace: ns, Name: name, Code: res.ActCode[i]})
		}
	}
	g0, g1 := groupRange(b.p, c)
	rec.Groups = res.Groups[g0:g1]
	for _, g := range rec.Groups {
		rec.CreateIdx = append(rec.CreateIdx, res.CreateIdx[g.create_off:g.create_off+g.n_create])
	}
	return rec
}

// groupRange reads c_group_off / c_group_cnt of the packed snapshot (kr_packer_bufs).
func groupRange(p *Packer, c uint32) (uint32, uint32) {
	var bufs C.kr_snapshot_bufs
	C.kr_packer_bufs(p.h, &bufs)
	cols := wrapColumns(&bufs, p.eng.sizes)
	return cols.CGroupOff[c], cols.CGroupOff[c] + cols.CGroupCnt[c]
}
