// kr_group_packer.cpp — the native packer sharded over GPUs (include/kr_engine.h kr_group_packer_*; DESIGN §6).  Host code on top
// of kr_packer (one per shard) and kr_group (the shards' worker threads, NUMA placement and the all-gather).
//
// Events are routed on the caller thread by the key (namespace, RayCluster name) — a RayCluster by its own, a Pod by its
// ray.io/cluster label, a RayJob by its cluster name — so a Pod always sits on the shard of every RayCluster its label can match
// (common/association.go:83-130): Pods never move when RayClusters come, go or are re-created under a new UID.  Only a relabelled
// Pod or a RayJob pointed at another cluster moves (deleted on its old shard, upserted on the new one).  flush / reconcile run on
// every shard's worker thread in parallel, each shard on its own incremental pipeline.
#include <functional>
#include <string>
#include <unordered_map>
#include <vector>

#include "../../include/kr_engine.h"

// kr_group.cpp
int kr_internal_group_create(const int32_t *devices, uint32_t n, const std::function<int(uint32_t, int, kr_engine **)> &make,
                             std::function<void(uint32_t, kr_engine *)> release, kr_group **out);
int kr_internal_group_run(kr_group *g, const std::function<int(uint32_t)> &f, uint32_t *failed_shard);
kr_sizes *kr_internal_group_sizes(kr_group *g, uint32_t i);
// kr_packer.cpp
extern "C" int64_t kr_internal_packer_find_pod(kr_packer *p, kr_str ns, kr_str name);

struct kr_group_packer {
  kr_group *g = nullptr;
  std::vector<kr_packer *> pk;
  std::unordered_map<std::string, uint32_t> job_shard;  // "ns\0name" -> the shard holding the RayJob (RayJobs are few)
  std::string err;
};

namespace {

uint32_t shard_of(const kr_group_packer *gp, kr_str ns, kr_str cluster) { return kr_shard_of_key(ns, cluster, (uint32_t)gp->pk.size()); }

int shard_fail(kr_group_packer *gp, uint32_t s, int rc) {
  gp->err = std::string("shard ") + std::to_string(s) + ": " + kr_packer_last_error(gp->pk[s]);
  return rc;
}

// every shard on its own worker thread, joined; the first failing shard's code and message
int run_all(kr_group_packer *gp, const std::function<int(uint32_t)> &f) {
  uint32_t bad = 0;
  gp->err.clear();
  const int rc = kr_internal_group_run(gp->g, f, &bad);
  return rc ? shard_fail(gp, bad, rc) : KR_OK;
}

std::string job_key(kr_str ns, kr_str name) {
  std::string k(ns.p, ns.n);
  k.push_back('\0');
  k.append(name.p, name.n);
  return k;
}

}  // namespace

extern "C" {

// FNV-1a 64 over ns + "/" + cluster_name, modulo n (the hash kr_packer_cluster_upsert stores as c_uid_hash for a RayCluster
// without a UID).  An absent name hashes like "".
uint32_t kr_shard_of_key(kr_str ns, kr_str cluster_name, uint32_t n) {
  if (n == 0) return 0;
  uint64_t h = 0xCBF29CE484222325ull;
  auto feed = [&h](const char *s, uint32_t k) { for (uint32_t i = 0; i < k; i++) { h ^= (uint8_t)s[i]; h *= 0x100000001B3ull; } };
  if (ns.p) feed(ns.p, ns.n);
  feed("/", 1);
  if (cluster_name.p) feed(cluster_name.p, cluster_name.n);
  return (uint32_t)(h % n);
}

int kr_group_packer_create(const kr_config *per_shard, const int32_t *devices, uint32_t n, kr_group_packer **out) {
  if (!per_shard || !out || n == 0 || n > 64) return KR_E_INVALID;
  *out = nullptr;
  kr_group_packer *gp = new kr_group_packer();
  gp->pk.assign(n, nullptr);
  const kr_config base = *per_shard;
  // each shard's packer (and so its engine and pinned arenas) is created on the shard's NUMA-bound worker thread; the group
  // frees each one there through kr_packer_destroy, which frees its engine
  int rc = kr_internal_group_create(devices, n, [gp, &base](uint32_t i, int device, kr_engine **e) {
    kr_config cfg = base;
    cfg.device = device;
    if (int r = kr_packer_create(&cfg, &gp->pk[i])) return r;
    *e = kr_packer_engine(gp->pk[i]);
    return (int)KR_OK;
  }, [gp](uint32_t i, kr_engine *) { kr_packer_destroy(gp->pk[i]); gp->pk[i] = nullptr; }, &gp->g);
  if (rc) { delete gp; return rc; }  // (kr_internal_group_create has destroyed the shards it made)
  *out = gp;
  return KR_OK;
}

void kr_group_packer_destroy(kr_group_packer *gp) {
  if (!gp) return;
  kr_group_destroy(gp->g);
  delete gp;
}

uint32_t kr_group_packer_size(kr_group_packer *gp) { return gp ? (uint32_t)gp->pk.size() : 0; }
kr_packer *kr_group_packer_shard(kr_group_packer *gp, uint32_t shard) { return (gp && shard < gp->pk.size()) ? gp->pk[shard] : nullptr; }
kr_group *kr_group_packer_group(kr_group_packer *gp) { return gp ? gp->g : nullptr; }
const char *kr_group_packer_last_error(kr_group_packer *gp) { return gp ? gp->err.c_str() : "null group packer"; }

// ---- events: on the caller thread, straight into the shard's packer
int kr_group_packer_pod_upsert(kr_group_packer *gp, const kr_pod_obj *o) {
  if (!gp || !o || !o->ns.p || !o->name.p) return KR_E_INVALID;
  const uint32_t n = (uint32_t)gp->pk.size(), s = shard_of(gp, o->ns, o->cluster);
  uint32_t old = s;  // a relabelled Pod still sits on the shard of its previous label
  if (n > 1 && kr_internal_packer_find_pod(gp->pk[s], o->ns, o->name) < 0)
    for (uint32_t j = 0; j < n; j++)
      if (j != s && kr_internal_packer_find_pod(gp->pk[j], o->ns, o->name) >= 0) { old = j; break; }
  if (int rc = kr_packer_pod_upsert(gp->pk[s], o)) return shard_fail(gp, s, rc);  // (on failure the Pod stays where it was)
  if (old != s)
    if (int rc = kr_packer_pod_delete(gp->pk[old], o->ns, o->name)) return shard_fail(gp, old, rc);
  return KR_OK;
}

int kr_group_packer_pod_delete(kr_group_packer *gp, kr_str ns, kr_str name) {
  if (!gp || !ns.p || !name.p) return KR_E_INVALID;
  for (uint32_t j = 0; j < gp->pk.size(); j++)
    if (kr_internal_packer_find_pod(gp->pk[j], ns, name) >= 0) {
      if (int rc = kr_packer_pod_delete(gp->pk[j], ns, name)) return shard_fail(gp, j, rc);
      return KR_OK;
    }
  return KR_OK;  // not in any shard: nothing to do
}

int kr_group_packer_cluster_upsert(kr_group_packer *gp, const kr_cluster_obj *o) {
  if (!gp || !o || !o->ns.p || !o->name.p) return KR_E_INVALID;
  const uint32_t s = shard_of(gp, o->ns, o->name);
  if (int rc = kr_packer_cluster_upsert(gp->pk[s], o)) return shard_fail(gp, s, rc);
  return KR_OK;
}

int kr_group_packer_cluster_delete(kr_group_packer *gp, kr_str ns, kr_str name) {
  if (!gp || !ns.p || !name.p) return KR_E_INVALID;
  const uint32_t s = shard_of(gp, ns, name);
  if (int rc = kr_packer_cluster_delete(gp->pk[s], ns, name)) return shard_fail(gp, s, rc);
  return KR_OK;
}

int kr_group_packer_job_upsert(kr_group_packer *gp, const kr_job_obj *o) {
  if (!gp || !o || !o->ns.p || !o->name.p) return KR_E_INVALID;
  const uint32_t s = shard_of(gp, o->ns, o->cluster_name);
  std::string key = job_key(o->ns, o->name);
  auto it = gp->job_shard.find(key);
  if (int rc = kr_packer_job_upsert(gp->pk[s], o)) return shard_fail(gp, s, rc);
  if (it == gp->job_shard.end()) { gp->job_shard.emplace(std::move(key), s); return KR_OK; }
  const uint32_t old = it->second;
  it->second = s;
  if (old != s)  // its cluster name moved it
    if (int rc = kr_packer_job_delete(gp->pk[old], o->ns, o->name)) return shard_fail(gp, old, rc);
  return KR_OK;
}

int kr_group_packer_job_delete(kr_group_packer *gp, kr_str ns, kr_str name) {
  if (!gp || !ns.p || !name.p) return KR_E_INVALID;
  auto it = gp->job_shard.find(job_key(ns, name));
  if (it == gp->job_shard.end()) return KR_OK;
  const uint32_t s = it->second;
  gp->job_shard.erase(it);
  if (int rc = kr_packer_job_delete(gp->pk[s], ns, name)) return shard_fail(gp, s, rc);
  return KR_OK;
}

// ---- epoch: every shard on its own worker thread
int kr_group_packer_flush(kr_group_packer *gp, uint32_t *modes_out) {
  if (!gp) return KR_E_INVALID;
  return run_all(gp, [gp, modes_out](uint32_t i) {
    uint32_t mode = 0;
    if (int rc = kr_packer_flush(gp->pk[i], &mode)) return rc;
    if (modes_out) modes_out[i] = mode;
    return kr_packer_sizes(gp->pk[i], kr_internal_group_sizes(gp->g, i));
  });
}

int kr_group_packer_reconcile(kr_group_packer *gp, const kr_flags *flags, kr_results_view *views) {
  if (!gp || !flags || !views) return KR_E_INVALID;
  return run_all(gp, [gp, flags, views](uint32_t i) { return kr_reconcile_batch(kr_packer_engine(gp->pk[i]), &flags[i], &views[i]); });
}

}  // extern "C"
