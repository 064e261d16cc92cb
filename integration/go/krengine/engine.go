package krengine

/*
#cgo CFLAGS: -I${SRCDIR}/../../../include
#cgo LDFLAGS: -L${SRCDIR}/../../../kuberay_b200 -lkrengine
#include <stdlib.h>
#include "kr_engine.h"
*/
import "C"

import (
	"errors"
	"fmt"
	"runtime"
	"unsafe"
)

// Sizes mirrors kr_sizes: the live row counts of one snapshot.
type Sizes struct {
	Clusters, Groups, Wtd, Pods, Heads, Jobs uint32
	JSONBytes                                uint64
}

func (n Sizes) c() C.kr_sizes {
	return C.kr_sizes{n_clusters: C.uint32_t(n.Clusters), n_groups: C.uint32_t(n.Groups), n_wtd: C.uint32_t(n.Wtd), n_pods: C.uint32_t(n.Pods),
		n_heads: C.uint32_t(n.Heads), n_jobs: C.uint32_t(n.Jobs), json_bytes: C.uint64_t(n.JSONBytes)}
}

// Config mirrors kr_config: device ordinal and arena capacities.
type Config struct {
	Device                                                                  int32
	MaxClusters, MaxGroups, MaxWtd, MaxPods, MaxHeads, MaxJobs, MaxCreates uint32
	MaxJSONBytes                                                            uint64
}

func (c Config) c() C.kr_config {
	return C.kr_config{device: C.int32_t(c.Device), max_clusters: C.uint32_t(c.MaxClusters), max_groups: C.uint32_t(c.MaxGroups), max_wtd: C.uint32_t(c.MaxWtd),
		max_pods: C.uint32_t(c.MaxPods), max_heads: C.uint32_t(c.MaxHeads), max_jobs: C.uint32_t(c.MaxJobs), max_creates: C.uint32_t(c.MaxCreates),
		max_json_bytes: C.uint64_t(c.MaxJSONBytes)}
}

// Flags mirrors kr_flags: the feature gates and environment switches reconcilePods / calculateStatus read, per pass.
type Flags struct {
	StatusConditionsGate bool   // features.RayClusterStatusConditions
	MultiHostIndexing    bool   // features.RayMultiHostIndexing
	RandomPodDelete      bool   // ENABLE_RANDOM_POD_DELETE
	SkipHash             bool   // test / bench knob: leave the digests out (the Recreate gate then treats them as unknown)
	FetchPodLists        bool   // false in production: compact action list only (bucket pipeline, incremental epochs)
	HeadNotFoundReason   uint32 // interned ids of the two HeadPodReady strings (kr_packer_intern)
	HeadNotFoundMessage  uint32
}

func b2u(b bool) C.uint8_t {
	if b {
		return 1
	}
	return 0
}

func (f Flags) c() C.kr_flags {
	return C.kr_flags{gate_status_conditions: b2u(f.StatusConditionsGate), gate_multihost_indexing: b2u(f.MultiHostIndexing), env_random_pod_delete: b2u(f.RandomPodDelete),
		skip_hash: b2u(f.SkipHash), fetch_pod_lists: b2u(f.FetchPodLists), id_head_not_found_reason: C.uint32_t(f.HeadNotFoundReason),
		id_head_not_found_msg: C.uint32_t(f.HeadNotFoundMessage)}
}

// Results are Go slices over the engine's pinned result arenas (valid until the next Begin / Reconcile on the same engine).
type Results struct {
	Clusters      []C.kr_cluster_result // [n_clusters] one record per RayCluster
	Hash          []byte                // [32*n_clusters] base32hex(sha1(muted spec JSON))
	Groups        []C.kr_group_result   // [n_groups]
	WtdPodIdx     []int32               // [n_wtd]
	CreateIdx     []int32               // [create_extent] replica indices; group g owns [create_off, create_off+n_create)
	Jobs          []C.kr_job_result     // [n_jobs]
	ActStart      []uint32              // [n_clusters+1]
	ActCnt        []uint32              // [n_clusters]
	ActPodIdx     []uint32              // [act_extent]
	ActCode       []uint8               // [act_extent] KR_ACT_*
	Changed       []uint32              // rows recomputed by an incremental epoch; nil after a full pass (every record is fresh)
	NCreateTotal  uint32
	NOrphans      uint32
	NActions      uint32
	NChanged      uint32
}

func wrapResults(v *C.kr_results_view, n Sizes) *Results {
	r := &Results{
		Clusters: unsafe.Slice((*C.kr_cluster_result)(unsafe.Pointer(v.clusters)), int(n.Clusters)),
		Hash:     unsafe.Slice((*byte)(unsafe.Pointer(v.hash)), int(n.Clusters)*32),
		Groups:   unsafe.Slice((*C.kr_group_result)(unsafe.Pointer(v.groups)), int(n.Groups)),
		WtdPodIdx: unsafe.Slice((*int32)(unsafe.Pointer(v.wtd_pod_idx)), int(n.Wtd)),
		CreateIdx: unsafe.Slice((*int32)(unsafe.Pointer(v.create_idx)), int(v.create_extent)),
		Jobs:      unsafe.Slice((*C.kr_job_result)(unsafe.Pointer(v.jobs)), int(n.Jobs)),
		ActStart:  unsafe.Slice((*uint32)(unsafe.Pointer(v.act_start)), int(n.Clusters)+1),
		ActCnt:    unsafe.Slice((*uint32)(unsafe.Pointer(v.act_cnt)), int(n.Clusters)),
		ActPodIdx: unsafe.Slice((*uint32)(unsafe.Pointer(v.act_pod_idx)), int(v.act_extent)),
		ActCode:   unsafe.Slice((*uint8)(unsafe.Pointer(v.act_code)), int(v.act_extent)),
		NCreateTotal: uint32(v.n_create_total), NOrphans: uint32(v.n_orphans), NActions: uint32(v.n_actions), NChanged: uint32(v.n_changed),
	}
	if v.changed_clusters != nil {
		r.Changed = unsafe.Slice((*uint32)(unsafe.Pointer(v.changed_clusters)), int(v.n_changed))
	}
	return r
}

// Engine is one kr_engine: one device, one snapshot resident at a time.  Not safe for concurrent use.
type Engine struct {
	h     *C.kr_engine
	sizes Sizes
	owned bool // false when the handle belongs to a Packer or a Group
}

// New creates an engine on cfg.Device.  It fails when no CUDA device is visible: there is no CPU fallback behind this boundary.
func New(cfg Config) (*Engine, error) {
	if C.kr_device_count() <= 0 {
		return nil, errors.New("krengine: no CUDA device visible")
	}
	cc := cfg.c()
	var h *C.kr_engine
	if rc := C.kr_engine_create(&cc, &h); rc != C.KR_OK {
		return nil, fmt.Errorf("krengine: kr_engine_create failed (%d)", int(rc))
	}
	return &Engine{h: h, owned: true}, nil
}

func (e *Engine) Close() {
	if e.owned && e.h != nil {
		C.kr_engine_destroy(e.h)
	}
	e.h = nil
}

func (e *Engine) err(rc C.int) error {
	return fmt.Errorf("krengine: %s (%d)", C.GoString(C.kr_last_error(e.h)), int(rc))
}

// Engine options (kr_engine_set_option).
const (
	OptFixedLayout   = uint32(C.KR_OPT_FIXED_LAYOUT)
	OptIncremental   = uint32(C.KR_OPT_INCREMENTAL)
	OptLargeClusters = uint32(C.KR_OPT_LARGE_CLUSTERS)
	OptWideClusters  = uint32(C.KR_OPT_WIDE_CLUSTERS)
	OptHugeClusters  = uint32(C.KR_OPT_HUGE_CLUSTERS)
	OptWtdEdits      = uint32(C.KR_OPT_WTD_EDITS)
	OptSpecRows      = uint32(C.KR_OPT_SPEC_ROWS)
	// OptClusterCreates is KR_OPT_CLUSTER_CREATES (1: RayClusters appended after the last row and RayJobs created or deleted keep
	// incremental epochs; only under KR_OPT_FIXED_LAYOUT; recommended for fleets that create RayClusters, such as RayJob and
	// RayService fleets; read at each Begin and object commit).
	OptClusterCreates = uint32(C.KR_OPT_CLUSTER_CREATES)
	// OptClusterDeletes is KR_OPT_CLUSTER_DELETES (1: RayClusters deleted by swap-remove keep incremental epochs; only under
	// KR_OPT_FIXED_LAYOUT; recommended for fleets that delete RayClusters, such as RayJob fleets with shutdownAfterJobFinishes;
	// read at each Begin and object commit).
	OptClusterDeletes = uint32(C.KR_OPT_CLUSTER_DELETES)
	// OptGroupEdits is KR_OPT_GROUP_EDITS (1: a RayCluster whose worker groups were appended, removed, renamed or reordered keeps
	// incremental epochs; only under KR_OPT_FIXED_LAYOUT; recommended for RayService fleets, whose in-place updates append worker
	// groups; read at each Begin and object commit).
	OptGroupEdits = uint32(C.KR_OPT_GROUP_EDITS)
	// OptLargeGrowth is KR_OPT_LARGE_GROWTH (1: a RayCluster that outgrows its bucket or region in an incremental epoch gets a new
	// region in that epoch; only with KR_OPT_LARGE_CLUSTERS; recommended for autoscaled fleets; read at each incremental pass).
	OptLargeGrowth = uint32(C.KR_OPT_LARGE_GROWTH)
	// OptLargeMoves is KR_OPT_LARGE_MOVES (1: KR_OPT_CLUSTER_DELETES and KR_OPT_GROUP_EDITS also keep incremental epochs when a large
	// RayCluster is deleted, moved by swap-remove or regrouped; only with KR_OPT_LARGE_CLUSTERS and KR_OPT_FIXED_LAYOUT; recommended
	// for RayJob fleets whose RayClusters grow large and RayService fleets; read at each object commit).
	OptLargeMoves = uint32(C.KR_OPT_LARGE_MOVES)
	// OptHugeGrowth is KR_OPT_HUGE_GROWTH (1: a RayCluster that grows past KR_LARGE_MAX_PODS Pods, or a huge one that outgrows its
	// region, in an incremental epoch gets a new region and tiles in that epoch; only with KR_OPT_LARGE_CLUSTERS, KR_OPT_HUGE_CLUSTERS
	// and KR_OPT_LARGE_GROWTH; recommended for fleets of very large autoscaled RayClusters; read at each incremental pass).
	OptHugeGrowth = uint32(C.KR_OPT_HUGE_GROWTH)
	// OptBucketPodLists is KR_OPT_BUCKET_POD_LISTS (1: FetchPodLists only asks for the full pod lists; the pass keeps its pipeline
	// and its incremental epoch, and the bucket pipeline builds the same lists and pod_start as the sort pipeline; for debug
	// endpoints and per-Pod logs on production fleets; read at each pass).
	OptBucketPodLists = uint32(C.KR_OPT_BUCKET_POD_LISTS)
	// OptJsonMoves is KR_OPT_JSON_MOVES (1, with KR_OPT_SPEC_ROWS: Packer.Flush commits a compaction of its JSON arena with
	// CommitJsonMoves instead of the whole arena and reports PackJsonMoves; recommended for RayJob fleets and spec rollouts, whose
	// dead spec bytes make the packer compact often; read by Packer.Flush).
	OptJsonMoves = uint32(C.KR_OPT_JSON_MOVES)
	// OptSMCount is KR_OPT_SM_COUNT (read only, with GetOption: the SM count the engine sizes its SM-sized grids by, the device's
	// multiprocessor count or the lower KR_SM_COUNT of the environment at New).
	OptSMCount = uint32(C.KR_OPT_SM_COUNT)
)

// SetOption: KR_OPT_FIXED_LAYOUT (before the first Begin), KR_OPT_INCREMENTAL, KR_OPT_LARGE_CLUSTERS (1: RayClusters of 257 to
// KR_LARGE_MAX_PODS pods stay on the bucket pipeline and keep incremental epochs; recommended for fleets that have them; takes
// effect at the next full pass), KR_OPT_WIDE_CLUSTERS (1: the same for RayClusters with more than 32 worker groups; takes effect
// at the next full pass), KR_OPT_HUGE_CLUSTERS (1, with KR_OPT_LARGE_CLUSTERS: the same for RayClusters of more than
// KR_LARGE_MAX_PODS pods; takes effect at the next full pass), KR_OPT_WTD_EDITS (1: scaleStrategy.workersToDelete edits keep
// incremental epochs; recommended for autoscaling fleets; read at each object commit), KR_OPT_SPEC_ROWS (1: Packer.Flush commits
// re-emitted specs with CommitSpecRows instead of the whole JSON arena and reports PackSpecRows), KR_OPT_CLUSTER_CREATES (1, with
// KR_OPT_FIXED_LAYOUT: RayClusters appended after the last row and RayJobs created or deleted keep incremental epochs; read at each
// Begin and object commit), KR_OPT_CLUSTER_DELETES (1, with KR_OPT_FIXED_LAYOUT: RayClusters deleted by swap-remove keep incremental
// epochs; read at each Begin and object commit), KR_OPT_GROUP_EDITS (1, with KR_OPT_FIXED_LAYOUT: a RayCluster whose list of worker
// groups changed keeps incremental epochs; read at each Begin and object commit), KR_OPT_LARGE_GROWTH (1, with KR_OPT_LARGE_CLUSTERS:
// a RayCluster that outgrows its bucket or region keeps incremental epochs; read at each incremental pass), KR_OPT_LARGE_MOVES (1, with
// KR_OPT_LARGE_CLUSTERS and KR_OPT_FIXED_LAYOUT: a large RayCluster deleted, moved or regrouped keeps incremental epochs; read at
// each object commit), KR_OPT_HUGE_GROWTH (1, with KR_OPT_LARGE_CLUSTERS, KR_OPT_HUGE_CLUSTERS and KR_OPT_LARGE_GROWTH: a RayCluster
// that grows past KR_LARGE_MAX_PODS Pods keeps incremental epochs; read at each incremental pass), KR_OPT_BUCKET_POD_LISTS (1:
// fetching the full pod lists keeps the pass's pipeline and its incremental epoch; read at each pass), KR_OPT_JSON_MOVES (1, with
// KR_OPT_SPEC_ROWS: Packer.Flush commits a compaction of its JSON arena with CommitJsonMoves and reports PackJsonMoves; read by
// Packer.Flush).  For a Packer, call it on Packer.Engine().
func (e *Engine) SetOption(option uint32, value uint64) error {
	if rc := C.kr_engine_set_option(e.h, C.uint32_t(option), C.uint64_t(value)); rc != C.KR_OK {
		return e.err(rc)
	}
	return nil
}

// GetOption reads an option's current value, or the read-only KR_OPT_SM_COUNT (kr_engine_get_option).
func (e *Engine) GetOption(option uint32) (uint64, error) {
	var v C.uint64_t
	if rc := C.kr_engine_get_option(e.h, C.uint32_t(option), &v); rc != C.KR_OK {
		return 0, e.err(rc)
	}
	return uint64(v), nil
}

// Begin hands out the pinned arenas for a snapshot of the given sizes.
func (e *Engine) Begin(n Sizes) (*Columns, error) {
	var bufs C.kr_snapshot_bufs
	sz := n.c()
	if rc := C.kr_snapshot_begin(e.h, &sz, &bufs); rc != C.KR_OK {
		return nil, e.err(rc)
	}
	e.sizes = n
	return wrapColumns(&bufs, n), nil
}

// Commit uploads the whole snapshot (asynchronously: it overlaps the previous pass' tail).
func (e *Engine) Commit() error {
	if rc := C.kr_snapshot_commit(e.h); rc != C.KR_OK {
		return e.err(rc)
	}
	return nil
}

// CommitParts uploads KR_PART_COLUMNS | KR_PART_JSON | KR_PART_OBJECTS.
func (e *Engine) CommitParts(parts uint32) error {
	if rc := C.kr_snapshot_commit_parts(e.h, C.uint32_t(parts)); rc != C.KR_OK {
		return e.err(rc)
	}
	return nil
}

// CommitPodRows uploads the pod rows rewritten in the arenas since the last epoch.  rows is ordinary Go memory without pointers:
// C copies it before returning.
func (e *Engine) CommitPodRows(rows []uint32) error {
	if len(rows) == 0 {
		return nil
	}
	if rc := C.kr_snapshot_commit_pod_rows(e.h, (*C.uint32_t)(unsafe.Pointer(&rows[0])), C.uint32_t(len(rows))); rc != C.KR_OK {
		return e.err(rc)
	}
	return nil
}

// CommitPodValues is the journal form: values[7*i+k] is pod column k of row rows[i] (rows distinct).
func (e *Engine) CommitPodValues(rows, values []uint32) error {
	if len(rows) == 0 {
		return nil
	}
	if len(values) != 7*len(rows) {
		return errors.New("krengine: CommitPodValues wants 7 values per row")
	}
	rc := C.kr_snapshot_commit_pod_values(e.h, (*C.uint32_t)(unsafe.Pointer(&rows[0])), (*C.uint32_t)(unsafe.Pointer(&values[0])), C.uint32_t(len(rows)))
	if rc != C.KR_OK {
		return e.err(rc)
	}
	return nil
}

// CommitObjectRows uploads only the RayCluster rows (with their groups) and head-aux rows that changed.
func (e *Engine) CommitObjectRows(clusterRows, headRows []uint32) error {
	var cp, hp *C.uint32_t
	if len(clusterRows) > 0 {
		cp = (*C.uint32_t)(unsafe.Pointer(&clusterRows[0]))
	}
	if len(headRows) > 0 {
		hp = (*C.uint32_t)(unsafe.Pointer(&headRows[0]))
	}
	if rc := C.kr_snapshot_commit_object_rows(e.h, cp, C.uint32_t(len(clusterRows)), hp, C.uint32_t(len(headRows))); rc != C.KR_OK {
		return e.err(rc)
	}
	return nil
}

// CommitSpecRows uploads only the muted-spec JSON ranges (and c_json_off / c_json_len) of the RayClusters whose spec was rewritten
// in the arenas; the next pass re-hashes only them.  Call it before CommitParts(KR_PART_OBJECTS) / CommitObjectRows; the arenas must
// not be rewritten until the next pass has returned.  clusterRows is ordinary Go memory without pointers: C copies it before returning.
func (e *Engine) CommitSpecRows(clusterRows []uint32) error {
	if len(clusterRows) == 0 {
		return nil
	}
	if rc := C.kr_snapshot_commit_spec_rows(e.h, (*C.uint32_t)(unsafe.Pointer(&clusterRows[0])), C.uint32_t(len(clusterRows))); rc != C.KR_OK {
		return e.err(rc)
	}
	return nil
}

// CommitJsonMoves tells the engine that the unchanged muted-spec JSON of these RayClusters now sits at the ranges c_json_off gives
// (same c_json_len), as after a compaction of the arena; the device moves its copies there, so no spec byte crosses PCIe and no
// digest is recomputed.  Call it before CommitSpecRows and the object commit of the epoch.  clusterRows is ordinary Go memory
// without pointers: C copies it before returning.
func (e *Engine) CommitJsonMoves(clusterRows []uint32) error {
	if len(clusterRows) == 0 {
		return nil
	}
	if rc := C.kr_snapshot_commit_json_moves(e.h, (*C.uint32_t)(unsafe.Pointer(&clusterRows[0])), C.uint32_t(len(clusterRows))); rc != C.KR_OK {
		return e.err(rc)
	}
	return nil
}

// Reconcile runs one pass (incremental on the device when the commits since the last pass allow it) and returns every record.
func (e *Engine) Reconcile(f Flags) (*Results, error) {
	var view C.kr_results_view
	cf := f.c()
	if rc := C.kr_reconcile_batch(e.h, &cf, &view); rc != C.KR_OK {
		return nil, e.err(rc) // the previous results are invalid now: the caller runs the per-object Go path for this epoch
	}
	return wrapResults(&view, e.sizes), nil
}

// PassReport is kr_pass_report: what the last pass was and why it was not an incremental epoch.
type PassReport struct {
	Incremental bool   // KR_PASSK_INCREMENTAL; false: a full pass
	Pipeline    uint8  // KR_PIPE_BUCKET / KR_PIPE_SORT / KR_PIPE_RADIX
	Attempts    uint8  // full-pass attempts that voided before the one that stood
	HashWait    bool   // a decide warp gave up waiting for its digest: the pass was rerun on the two-phase schedule
	Stride      uint32 // bucket stride; 0 off the bucket pipeline
	WhyFull     uint32 // KR_FULL_* bits; 0 for an incremental pass
}

// FullCauses names the KR_FULL_* bits, in bit order: the label values of an operator's per-cause counter.
var FullCauses = []struct {
	Bit  uint32
	Name string
}{
	{C.KR_FULL_FIRST, "first"}, {C.KR_FULL_CAPACITY, "capacity"}, {C.KR_FULL_DISABLED, "disabled"}, {C.KR_FULL_FLAGS, "flags"},
	{C.KR_FULL_POD_LISTS, "pod_lists"}, {C.KR_FULL_LARGE, "large"}, {C.KR_FULL_WIDE, "wide"}, {C.KR_FULL_OPTION, "option"},
	{C.KR_FULL_COLUMNS, "columns"}, {C.KR_FULL_SIZES, "sizes"}, {C.KR_FULL_STRUCTURAL, "structural"}, {C.KR_FULL_ROW_MAP, "row_map"},
	{C.KR_FULL_OVERFLOW, "overflow"}, {C.KR_FULL_GROW_LIMIT, "grow_limit"}, {C.KR_FULL_ARENA, "arena"},
	{C.KR_FULL_EPOCH_WRAP, "epoch_wrap"},
}

// LastPass reports the last pass that returned KR_OK (one struct copy, no device work).
func (e *Engine) LastPass() (PassReport, error) {
	var r C.kr_pass_report
	if rc := C.kr_last_pass(e.h, &r); rc != C.KR_OK {
		return PassReport{}, e.err(rc)
	}
	return PassReport{Incremental: r.kind == C.KR_PASSK_INCREMENTAL, Pipeline: uint8(r.pipeline), Attempts: uint8(r.attempts),
		HashWait: r.hash_wait != 0, Stride: uint32(r.stride), WhyFull: uint32(r.why_full)}, nil
}

// HashBatch: utils.GenerateJsonHash's digest half for n messages (msgs[offsets[i]:offsets[i+1]]); out receives 32 characters each.
func (e *Engine) HashBatch(msgs []byte, offsets []uint64, out []byte) error {
	n := len(offsets) - 1
	if n <= 0 {
		return nil
	}
	if len(out) < 32*n {
		return errors.New("krengine: HashBatch output too small")
	}
	var mp *C.uint8_t
	if len(msgs) > 0 {
		mp = (*C.uint8_t)(unsafe.Pointer(&msgs[0]))
	}
	rc := C.kr_hash_batch(e.h, mp, (*C.uint64_t)(unsafe.Pointer(&offsets[0])), C.uint32_t(n), (*C.char)(unsafe.Pointer(&out[0])))
	if rc != C.KR_OK {
		return e.err(rc)
	}
	return nil
}

// HashCompareRow is one isClusterSpecHashEqual question (rayservice_controller.go:1130-1157).
type HashCompareRow struct {
	GoalSpecJSON    []byte // json.Marshal(rayService.Spec.RayClusterSpec), any key order
	ClusterHash     string // the RayCluster's ray.io/hash-without-replicas-and-workers-to-delete annotation
	NumWorkerGroups string // its ray.io/num-worker-groups annotation (read only when Partial)
	Partial         bool
}

// HashCompare answers a batch of them: mute + marshal on host threads, one SHA-1 launch, compare.
func (e *Engine) HashCompare(rows []HashCompareRow) ([]bool, error) {
	if len(rows) == 0 {
		return nil, nil
	}
	var s strs
	defer s.release()
	cr := make([]C.kr_hash_compare_row, len(rows))
	for i := range rows {
		r := &rows[i]
		if len(r.GoalSpecJSON) > 0 {
			s.pin.Pin(&r.GoalSpecJSON[0])
			cr[i].goal_spec_json = (*C.uint8_t)(unsafe.Pointer(&r.GoalSpecJSON[0]))
			cr[i].goal_spec_len = C.uint64_t(len(r.GoalSpecJSON))
		}
		h, w := s.str(r.ClusterHash), s.str(r.NumWorkerGroups)
		cr[i].cluster_hash, cr[i].cluster_hash_len = h.p, h.n
		cr[i].num_worker_groups, cr[i].num_worker_groups_len = w.p, w.n
		cr[i].partial = b2u(r.Partial)
	}
	eq := make([]uint8, len(rows))
	rc := C.kr_hash_compare_batch(e.h, &cr[0], C.uint32_t(len(rows)), (*C.uint8_t)(unsafe.Pointer(&eq[0])), nil)
	if rc != C.KR_OK {
		return nil, e.err(rc)
	}
	out := make([]bool, len(rows))
	for i, v := range eq {
		out[i] = v != 0
	}
	return out, nil
}

// strs builds kr_str values that point into Go strings and keeps those strings pinned until release(): cgo allows a pinned Go pointer
// inside memory passed to C (runtime.Pinner, Go 1.21).
type strs struct{ pin runtime.Pinner }

// str: "" becomes the ABSENT kr_str (p == NULL).
func (s *strs) str(v string) C.kr_str {
	if v == "" {
		return C.kr_str{}
	}
	p := unsafe.StringData(v)
	s.pin.Pin(p)
	return C.kr_str{p: (*C.char)(unsafe.Pointer(p)), n: C.uint32_t(len(v))}
}

var emptyByte = [1]byte{0}

// present: a string that is there even when empty (an annotation set to ""): p != NULL, n == 0.
func (s *strs) present(v string) C.kr_str {
	if v == "" {
		s.pin.Pin(&emptyByte[0])
		return C.kr_str{p: (*C.char)(unsafe.Pointer(&emptyByte[0])), n: 0}
	}
	return s.str(v)
}

// opt: nil -> absent, else present.
func (s *strs) opt(v *string) C.kr_str {
	if v == nil {
		return C.kr_str{}
	}
	return s.present(*v)
}

func (s *strs) bytes(b []byte) C.kr_str {
	if len(b) == 0 {
		return C.kr_str{}
	}
	s.pin.Pin(&b[0])
	return C.kr_str{p: (*C.char)(unsafe.Pointer(&b[0])), n: C.uint32_t(len(b))}
}

func (s *strs) release() { s.pin.Unpin() }
