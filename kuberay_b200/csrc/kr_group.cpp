// kr_group.cpp — multi-GPU coordinator of the reconcile engine (include/kr_engine.h kr_group_*; SURVEY §8(b) "one engine per device +
// a coordinator", §8(e)).  Host code on top of the single-device C ABI.
//
// A RayCluster's decisions depend only on its own spec, groups and pods (common/association.go:83-130): the snapshot shards by
// cluster-UID hash with NO data-path collective.  The coordinator owns one engine per shard, each driven by its own host thread
// pinned to the GPU's NUMA node (the thread also creates the engine, so the pinned arenas are allocated node-local: eight
// concurrent 66 MB uploads out of remote memory were what bent the round-1 e2e scaling curve), and offers
//   * kr_group_route: native UID-hash routing of a global snapshot into the shards' pinned arenas — clusters by
//     uid_hash64 % n, pods through the (namespace, ray.io/cluster) -> cluster table, orphans by a hash of their key, RayJobs
//     after their RayCluster — with every index column (g_cluster_idx, c_group_off, g_wtd_off, h_pod_idx) rewritten;
//   * kr_group_commit / kr_group_reconcile: every shard in parallel;
//   * kr_group_allgather_group_results: the optional exchange step of §8(e) — every device receives every shard's per-group
//     delta records (kr_group_result, 32 B each) — over NCCL (ncclAllGather issued from the coordinator thread, one
//     communicator per device; the library is looked up at run time) when every shard sits on its own device, by peer
//     copies otherwise (several shards on one GPU: tests on a single-GPU box).
// The worker threads, NUMA placement and exchange are shared with the group packer (kr_group_packer.cpp): its shards are
// kr_packers, made on the same workers by kr_internal_group_create, and the group frees each engine through its owner.
#include <cuda_runtime.h>
#include <dlfcn.h>
#include <sched.h>

#include <algorithm>
#include <condition_variable>
#include <cstdio>
#include <cstring>
#include <functional>
#include <mutex>
#include <string>
#include <thread>
#include <unordered_map>
#include <vector>

#include "../../include/kr_engine.h"

namespace {

// ---------------------------------------------------------------------------------------------- NUMA placement
std::vector<int> cpus_of_device(int device) {
  std::vector<int> cpus;
  char bus[32] = {0};
  if (cudaDeviceGetPCIBusId(bus, sizeof bus, device) != cudaSuccess) { cudaGetLastError(); return cpus; }
  for (char *p = bus; *p; p++) if (*p >= 'A' && *p <= 'Z') *p = (char)(*p - 'A' + 'a');
  char path[256];
  snprintf(path, sizeof path, "/sys/bus/pci/devices/%s/numa_node", bus);
  int node = -1;
  if (FILE *f = fopen(path, "r")) { if (fscanf(f, "%d", &node) != 1) node = -1; fclose(f); }
  if (node < 0) return cpus;
  snprintf(path, sizeof path, "/sys/devices/system/node/node%d/cpulist", node);
  if (FILE *f = fopen(path, "r")) {
    int a, b;
    char sep;
    while (fscanf(f, "%d", &a) == 1) {
      b = a;
      if (fscanf(f, "%c", &sep) == 1 && sep == '-') { if (fscanf(f, "%d", &b) != 1) b = a; if (fscanf(f, "%c", &sep) != 1) sep = 0; }
      for (int c = a; c <= b; c++) cpus.push_back(c);
      if (sep != ',') break;
    }
    fclose(f);
  }
  return cpus;
}

// ---------------------------------------------------------------------------------------------- one worker thread per shard
struct Worker {
  std::thread th;
  std::mutex mu;
  std::condition_variable cv;
  std::function<void()> job;
  bool has_job = false, done = true, quit = false;
  void start(int device) {
    th = std::thread([this, device] {
      std::vector<int> cpus = cpus_of_device(device);
      if (!cpus.empty()) {
        cpu_set_t set;
        CPU_ZERO(&set);
        for (int c : cpus) if (c < CPU_SETSIZE) CPU_SET(c, &set);
        sched_setaffinity(0, sizeof set, &set);  // best effort: a restricted cgroup keeps what it allows
      }
      cudaSetDevice(device);
      std::unique_lock<std::mutex> lk(mu);
      while (true) {
        cv.wait(lk, [this] { return has_job || quit; });
        if (quit) return;
        auto j = std::move(job);
        has_job = false;
        lk.unlock();
        j();
        lk.lock();
        done = true;
        cv.notify_all();
      }
    });
  }
  void submit(std::function<void()> j) {
    std::lock_guard<std::mutex> lk(mu);
    job = std::move(j); has_job = true; done = false;
    cv.notify_all();
  }
  void wait() { std::unique_lock<std::mutex> lk(mu); cv.wait(lk, [this] { return done; }); }
  void stop() {
    { std::lock_guard<std::mutex> lk(mu); quit = true; }
    cv.notify_all();
    if (th.joinable()) th.join();
  }
};

// ---------------------------------------------------------------------------------------------- NCCL, looked up at run time
typedef struct ncclComm *ncclComm_t;
struct Nccl {
  void *h = nullptr;
  int (*CommInitAll)(ncclComm_t *, int, const int *) = nullptr;
  int (*CommDestroy)(ncclComm_t) = nullptr;
  int (*GroupStart)() = nullptr;
  int (*GroupEnd)() = nullptr;
  int (*AllGather)(const void *, void *, size_t, int, ncclComm_t, cudaStream_t) = nullptr;
  bool load() {
    for (const char *name : {"libnccl.so.2", "libnccl.so"}) {
      h = dlopen(name, RTLD_NOW | RTLD_GLOBAL);
      if (h) break;
    }
    if (!h) return false;
    CommInitAll = (decltype(CommInitAll))dlsym(h, "ncclCommInitAll");
    CommDestroy = (decltype(CommDestroy))dlsym(h, "ncclCommDestroy");
    GroupStart = (decltype(GroupStart))dlsym(h, "ncclGroupStart");
    GroupEnd = (decltype(GroupEnd))dlsym(h, "ncclGroupEnd");
    AllGather = (decltype(AllGather))dlsym(h, "ncclAllGather");
    return CommInitAll && CommDestroy && GroupStart && GroupEnd && AllGather;
  }
};

inline uint64_t splitmix64(uint64_t x) {
  x += 0x9E3779B97F4A7C15ull;
  uint64_t z = x;
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return z ^ (z >> 31);
}

}  // namespace

struct kr_group {
  std::vector<kr_engine *> eng;
  std::vector<int> device;
  std::vector<Worker *> worker;
  std::vector<kr_snapshot_bufs> bufs;     // the shards' pinned arenas after kr_group_route / kr_group_begin
  std::vector<kr_sizes> sizes;
  std::vector<int> rc;
  std::string err;
  bool distinct_devices = true;
  std::function<void(uint32_t, kr_engine *)> release;  // frees shard i's engine (kr_group_create: kr_engine_destroy; a group packer: its kr_packer)
  // exchange step
  Nccl nccl;
  bool nccl_tried = false, nccl_ok = false;
  std::vector<ncclComm_t> comm;
  std::vector<cudaStream_t> xstream;
  std::vector<uint8_t *> xsend, xrecv;
  uint64_t xcap = 0;  // bytes per shard slot
};

namespace {

int gfail(kr_group *g, int code, const std::string &m) { if (g) g->err = m; return code; }

}  // namespace

// Shared with kr_group_packer.cpp: f(i) on shard i's thread, all joined; returns the first failing code and its shard.
int kr_internal_group_run(kr_group *g, const std::function<int(uint32_t)> &f, uint32_t *failed_shard) {
  const size_t n = g->eng.size();
  for (size_t i = 0; i < n; i++) g->worker[i]->submit([g, i, &f] { g->rc[i] = f((uint32_t)i); });
  for (size_t i = 0; i < n; i++) g->worker[i]->wait();
  for (size_t i = 0; i < n; i++)
    if (g->rc[i]) { if (failed_shard) *failed_shard = (uint32_t)i; return g->rc[i]; }
  return KR_OK;
}

// One worker thread per shard (pinned to its device's NUMA node), and on it make(i, device, &engine): whatever owns the engine is
// created there, so its pinned arenas are node-local.  kr_group_destroy calls release(i, engine) on the same thread for every shard
// that got an engine — the engine is freed there and nowhere else.
int kr_internal_group_create(const int32_t *devices, uint32_t n, const std::function<int(uint32_t, int, kr_engine **)> &make,
                             std::function<void(uint32_t, kr_engine *)> release, kr_group **out) {
  if (!out || n == 0 || n > 64) return KR_E_INVALID;
  *out = nullptr;
  int ndev = kr_device_count();
  if (ndev <= 0) return KR_E_NO_DEVICE;
  kr_group *g = new kr_group();
  g->release = std::move(release);
  g->eng.assign(n, nullptr); g->device.resize(n); g->rc.assign(n, 0); g->bufs.resize(n); g->sizes.resize(n);
  for (uint32_t i = 0; i < n; i++) {
    g->device[i] = devices ? devices[i] : (int)(i % (uint32_t)ndev);
    if (g->device[i] < 0 || g->device[i] >= ndev) { delete g; return KR_E_INVALID; }
    for (uint32_t j = 0; j < i; j++) if (g->device[j] == g->device[i]) g->distinct_devices = false;
  }
  for (uint32_t i = 0; i < n; i++) { g->worker.push_back(new Worker()); g->worker[i]->start(g->device[i]); }
  int rc = kr_internal_group_run(g, [g, &make](uint32_t i) { return make(i, g->device[i], &g->eng[i]); }, nullptr);
  if (rc) { kr_group_destroy(g); return rc; }
  *out = g;
  return KR_OK;
}

// The live row counts of shard i (kr_group_allgather_group_results sizes its slots by them): kr_group_route sets them, a group
// packer after each flush.
kr_sizes *kr_internal_group_sizes(kr_group *g, uint32_t i) { return &g->sizes[i]; }

namespace {

template <class F>
int for_all(kr_group *g, F f) {  // f(i) on shard i's thread; first failing code wins
  uint32_t bad = 0;
  const int rc = kr_internal_group_run(g, f, &bad);
  if (rc) g->err = std::string("shard ") + std::to_string(bad) + ": " + kr_last_error(g->eng[bad]);
  return rc;
}

}  // namespace

extern "C" {

int kr_group_create(const kr_config *per_shard, const int32_t *devices, uint32_t n, kr_group **out) {
  if (!per_shard) return KR_E_INVALID;
  const kr_config base = *per_shard;
  return kr_internal_group_create(devices, n, [&base](uint32_t, int device, kr_engine **e) {
    kr_config cfg = base;
    cfg.device = device;
    return kr_engine_create(&cfg, e);
  }, [](uint32_t, kr_engine *e) { kr_engine_destroy(e); }, out);
}

void kr_group_destroy(kr_group *g) {
  if (!g) return;
  for (size_t i = 0; i < g->eng.size(); i++) {
    if (i < g->worker.size()) {
      g->worker[i]->submit([g, i] {
        if (i < g->comm.size() && g->comm[i] && g->nccl.CommDestroy) g->nccl.CommDestroy(g->comm[i]);
        if (i < g->xstream.size() && g->xstream[i]) cudaStreamDestroy(g->xstream[i]);
        if (i < g->xsend.size() && g->xsend[i]) cudaFree(g->xsend[i]);
        if (i < g->xrecv.size() && g->xrecv[i]) cudaFree(g->xrecv[i]);
        if (g->eng[i]) g->release((uint32_t)i, g->eng[i]);
        g->rc[i] = 0;
      });
      g->worker[i]->wait();
    }
  }
  for (Worker *w : g->worker) { w->stop(); delete w; }
  delete g;
}

uint32_t kr_group_size(kr_group *g) { return g ? (uint32_t)g->eng.size() : 0; }
kr_engine *kr_group_engine(kr_group *g, uint32_t i) { return (g && i < g->eng.size()) ? g->eng[i] : nullptr; }
int kr_group_device(kr_group *g, uint32_t i) { return (g && i < g->device.size()) ? g->device[i] : -1; }
const char *kr_group_last_error(kr_group *g) { return g ? g->err.c_str() : "null group"; }
uint32_t kr_group_shard_of_uid(kr_group *g, uint64_t uid_hash) { return g && !g->eng.empty() ? (uint32_t)(uid_hash % g->eng.size()) : 0; }

// Route a global snapshot (host columns `in`, sizes `n`) into the shards: begin + fill of every engine.  shard_sizes_out[i]
// (optional) receives each shard's row counts; pod_shard_out / pod_row_out (optional, [n_pods]) say where every global pod row
// went, cluster_shard_out / cluster_row_out ([n_clusters]) likewise — the shim maps result rows back through them.
int kr_group_route(kr_group *g, const kr_snapshot_bufs *in, const kr_sizes *n, kr_sizes *shard_sizes_out, uint32_t *cluster_shard_out, uint32_t *cluster_row_out,
                   uint32_t *pod_shard_out, uint32_t *pod_row_out) {
  if (!g || !in || !n) return KR_E_INVALID;
  const uint32_t W = (uint32_t)g->eng.size();
  const uint32_t Nc = n->n_clusters, Ng = n->n_groups, Np = n->n_pods, Nh = n->n_heads, Nj = n->n_jobs;
  // clusters -> shard (uid_hash64 % W); (ns, name) -> cluster for the pods and the RayJobs
  std::vector<uint32_t> c_shard(Nc), c_row(Nc);
  std::vector<kr_sizes> sz(W);
  for (auto &s : sz) memset(&s, 0, sizeof s);
  std::unordered_map<uint64_t, uint32_t> by_key;
  by_key.reserve((size_t)Nc * 2 + 16);
  for (uint32_t c = 0; c < Nc; c++) {
    const uint32_t s = (uint32_t)(in->c_uid_hash[c] % W);
    c_shard[c] = s; c_row[c] = sz[s].n_clusters++;
    by_key.emplace(((uint64_t)in->c_ns_id[c] << 32) | in->c_name_id[c], c);  // duplicates: the lowest index wins (emplace keeps the first)
    sz[s].n_groups += in->c_group_cnt[c];
    sz[s].json_bytes += ((uint64_t)in->c_json_len[c] + 15) & ~15ull;
  }
  for (uint32_t gi = 0; gi < Ng; gi++) sz[c_shard[in->g_cluster_idx[gi]]].n_wtd += in->g_wtd_cnt[gi];
  std::vector<uint32_t> p_shard(Np), p_row(Np);
  for (uint32_t p = 0; p < Np; p++) {
    const uint64_t key = ((uint64_t)in->p_ns_id[p] << 32) | in->p_cluster_name_id[p];
    auto it = in->p_cluster_name_id[p] ? by_key.find(key) : by_key.end();
    const uint32_t s = it != by_key.end() ? c_shard[it->second] : (uint32_t)(splitmix64(key) % W);
    p_shard[p] = s; p_row[p] = sz[s].n_pods++;
  }
  for (uint32_t h = 0; h < Nh; h++) { if (in->h_pod_idx[h] >= Np) return gfail(g, KR_E_INVALID, "kr_group_route: h_pod_idx out of range"); sz[p_shard[in->h_pod_idx[h]]].n_heads++; }
  std::vector<uint32_t> j_shard(Nj);
  for (uint32_t j = 0; j < Nj; j++) {
    const uint64_t key = ((uint64_t)in->j_ns_id[j] << 32) | in->j_cluster_name_id[j];
    auto it = by_key.find(key);
    j_shard[j] = it != by_key.end() ? c_shard[it->second] : (uint32_t)(splitmix64(key) % W);
    sz[j_shard[j]].n_jobs++;
  }
  // begin every shard (its own thread: the engine's device is current there)
  g->sizes = sz;
  int rc = for_all(g, [g](uint32_t i) { return kr_snapshot_begin(g->eng[i], &g->sizes[i], &g->bufs[i]); });
  if (rc) return rc;
  // fill: one pass per table, rows appended in global order (List order is preserved inside every shard)
  std::vector<uint32_t> cg(W, 0), cw(W, 0), ch(W, 0), cj(W, 0);
  std::vector<uint64_t> cjs(W, 0);
  for (uint32_t c = 0; c < Nc; c++) {
    const uint32_t s = c_shard[c], r = c_row[c];
    kr_snapshot_bufs &o = g->bufs[s];
#define CP1(f) o.f[r] = in->f[c]
#define CPN(f, k) memcpy(&o.f[(size_t)(k) * r], &in->f[(size_t)(k) * c], sizeof(o.f[0]) * (k))
    CP1(c_ns_id); CP1(c_name_id); CP1(c_uid_hash); CP1(c_flags); CP1(c_suspend_status); CP1(c_ext_err_kind); CP1(c_ext_err_msg_id);
    CP1(c_group_cnt); CP1(c_json_len); CP1(c_old_state); CPN(c_old_counts, 5); CPN(c_old_cond_status, 5); CPN(c_old_cond_variant, 5);
    CP1(c_old_cond_reason_id); CPN(c_old_cond_msg_id, 2); CPN(c_old_head_ids, 4); CP1(c_svc_count); CP1(c_svc_ip_kind); CP1(c_svc_ip_id);
    CP1(c_svc_name_id); CP1(c_summary_id);
#undef CP1
#undef CPN
    o.c_group_off[r] = cg[s];
    o.c_json_off[r] = cjs[s];
    const uint64_t len = in->c_json_len[c], padded = (len + 15) & ~15ull;
    memcpy(o.json + cjs[s], in->json + in->c_json_off[c], len);
    if (padded > len) memset(o.json + cjs[s] + len, 0, padded - len);
    cjs[s] += padded;
    for (uint32_t k = 0; k < in->c_group_cnt[c]; k++) {
      const uint32_t gi = in->c_group_off[c] + k, go = cg[s]++;
      o.g_cluster_idx[go] = r; o.g_name_id[go] = in->g_name_id[gi]; o.g_replicas[go] = in->g_replicas[gi]; o.g_min[go] = in->g_min[gi];
      o.g_max[go] = in->g_max[gi]; o.g_num_hosts[go] = in->g_num_hosts[gi]; o.g_flags[go] = in->g_flags[gi];
      o.g_wtd_off[go] = cw[s]; o.g_wtd_cnt[go] = in->g_wtd_cnt[gi];
      for (uint32_t w = 0; w < in->g_wtd_cnt[gi]; w++) o.w_name_id[cw[s]++] = in->w_name_id[in->g_wtd_off[gi] + w];
    }
  }
  for (uint32_t p = 0; p < Np; p++) {
    kr_snapshot_bufs &o = g->bufs[p_shard[p]];
    const uint32_t r = p_row[p];
    o.p_ns_id[r] = in->p_ns_id[p]; o.p_cluster_name_id[r] = in->p_cluster_name_id[p]; o.p_group_name_id[r] = in->p_group_name_id[p];
    o.p_name_id[r] = in->p_name_id[p]; o.p_packed[r] = in->p_packed[p]; o.p_replica_index[r] = in->p_replica_index[p];
    o.p_replica_name_id[r] = in->p_replica_name_id[p];
  }
  for (uint32_t h = 0; h < Nh; h++) {
    const uint32_t p = in->h_pod_idx[h], s = p_shard[p], r = ch[s]++;
    kr_snapshot_bufs &o = g->bufs[s];
    o.h_pod_idx[r] = p_row[p]; o.h_ready_status[r] = in->h_ready_status[h]; o.h_ready_reason_id[r] = in->h_ready_reason_id[h];
    o.h_ready_msg_id[r] = in->h_ready_msg_id[h]; o.h_pod_ip_id[r] = in->h_pod_ip_id[h]; o.h_annot_state[r] = in->h_annot_state[h];
    o.h_version_state[r] = in->h_version_state[h];
    memcpy(o.h_annot_hash + 32 * (size_t)r, in->h_annot_hash + 32 * (size_t)h, 32);
  }
  for (uint32_t j = 0; j < Nj; j++) {
    const uint32_t s = j_shard[j], r = cj[s]++;
    kr_snapshot_bufs &o = g->bufs[s];
    o.j_ns_id[r] = in->j_ns_id[j]; o.j_cluster_name_id[r] = in->j_cluster_name_id[j]; o.j_summary_id[r] = in->j_summary_id[j];
  }
  if (shard_sizes_out) memcpy(shard_sizes_out, sz.data(), sizeof(kr_sizes) * W);
  if (cluster_shard_out) memcpy(cluster_shard_out, c_shard.data(), 4 * (size_t)Nc);
  if (cluster_row_out) memcpy(cluster_row_out, c_row.data(), 4 * (size_t)Nc);
  if (pod_shard_out) memcpy(pod_shard_out, p_shard.data(), 4 * (size_t)Np);
  if (pod_row_out) memcpy(pod_row_out, p_row.data(), 4 * (size_t)Np);
  return KR_OK;
}

int kr_group_commit(kr_group *g, uint32_t parts) {
  if (!g) return KR_E_INVALID;
  return for_all(g, [g, parts](uint32_t i) { return kr_snapshot_commit_parts(g->eng[i], parts); });
}

int kr_group_reconcile(kr_group *g, const kr_flags *flags, kr_results_view *views) {
  if (!g || !flags || !views) return KR_E_INVALID;
  const kr_flags f = *flags;
  return for_all(g, [g, f, views](uint32_t i) { return kr_reconcile_batch(g->eng[i], &f, &views[i]); });
}

// The optional exchange step (SURVEY §8(e)): after a pass, every device receives every shard's per-group delta records.
// slot_bytes = 32 * (largest shard's n_groups); the gathered buffer of device i holds n slots of slot_bytes, slot j = shard j's
// records (zero padded).  host_out (optional) receives device 0's gathered copy.  used_nccl_out: 1 NCCL, 0 peer copies.
int kr_group_allgather_group_results(kr_group *g, void *host_out, uint64_t host_cap, uint64_t *slot_bytes_out, int *used_nccl_out) {
  if (!g) return KR_E_INVALID;
  const uint32_t W = (uint32_t)g->eng.size();
  uint64_t slot = 0;
  for (uint32_t i = 0; i < W; i++) slot = std::max<uint64_t>(slot, 32ull * g->sizes[i].n_groups);
  slot = (slot + 255) & ~255ull;
  if (slot_bytes_out) *slot_bytes_out = slot;
  if (host_out && host_cap < slot * W) return gfail(g, KR_E_CAPACITY, "kr_group_allgather_group_results: host buffer too small");
  if (slot == 0) return KR_OK;
  if (g->xsend.empty()) { g->xsend.assign(W, nullptr); g->xrecv.assign(W, nullptr); g->xstream.assign(W, nullptr); g->comm.assign(W, nullptr); }
  if (slot > g->xcap) {
    g->xcap = slot + slot / 4;
    int rc = for_all(g, [g, W](uint32_t i) {
      if (g->xsend[i]) cudaFree(g->xsend[i]);
      if (g->xrecv[i]) cudaFree(g->xrecv[i]);
      if (!g->xstream[i] && cudaStreamCreateWithFlags(&g->xstream[i], cudaStreamNonBlocking) != cudaSuccess) return (int)KR_E_CUDA;
      if (cudaMalloc((void **)&g->xsend[i], g->xcap) != cudaSuccess || cudaMalloc((void **)&g->xrecv[i], g->xcap * W) != cudaSuccess) return (int)KR_E_CUDA;
      return (int)KR_OK;
    });
    if (rc) return rc;
  }
  if (!g->nccl_tried) {
    g->nccl_tried = true;
    if (g->distinct_devices && W > 1 && g->nccl.load()) {
      std::vector<int> devs(g->device.begin(), g->device.end());
      g->nccl_ok = g->nccl.CommInitAll(g->comm.data(), (int)W, devs.data()) == 0;  // from the coordinator thread, as §8(b) asks
    }
  }
  // stage every shard's records into its send slot (device-to-device on the shard's own device)
  int rc = for_all(g, [g, slot](uint32_t i) {
    if (cudaMemsetAsync(g->xsend[i], 0, slot, g->xstream[i]) != cudaSuccess) return (int)KR_E_CUDA;
    cudaStreamSynchronize(g->xstream[i]);
    return kr_group_results_copy(g->eng[i], g->xsend[i], 32ull * g->sizes[i].n_groups);
  });
  if (rc) return rc;
  if (g->nccl_ok) {
    g->nccl.GroupStart();
    for (uint32_t i = 0; i < W; i++) g->nccl.AllGather(g->xsend[i], g->xrecv[i], slot, /*ncclInt8*/ 0, g->comm[i], g->xstream[i]);
    if (g->nccl.GroupEnd() != 0) return gfail(g, KR_E_CUDA, "ncclAllGather failed");
    for (uint32_t i = 0; i < W; i++) { cudaSetDevice(g->device[i]); cudaStreamSynchronize(g->xstream[i]); }
  } else {
    for (uint32_t i = 0; i < W; i++)
      for (uint32_t j = 0; j < W; j++)
        if (cudaMemcpyPeerAsync(g->xrecv[i] + slot * j, g->device[i], g->xsend[j], g->device[j], slot, g->xstream[i]) != cudaSuccess)
          return gfail(g, KR_E_CUDA, "cudaMemcpyPeerAsync failed");
    for (uint32_t i = 0; i < W; i++) { cudaSetDevice(g->device[i]); cudaStreamSynchronize(g->xstream[i]); }
  }
  if (used_nccl_out) *used_nccl_out = g->nccl_ok ? 1 : 0;
  if (host_out) {
    cudaSetDevice(g->device[0]);
    if (cudaMemcpy(host_out, g->xrecv[0], slot * W, cudaMemcpyDeviceToHost) != cudaSuccess) return gfail(g, KR_E_CUDA, "gather download failed");
  }
  return KR_OK;
}

}  // extern "C"
