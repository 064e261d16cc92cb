/*
 * kr_oracle.c — CPU restatement of KubeRay's reconcilePods()/calculateStatus() decision logic.
 * TEST INFRASTRUCTURE ONLY — see kr_oracle.h for the scope, the reference citations and the pinning status.
 *
 * Each function cites the reference lines it follows (paths relative to ray-operator/controllers/ray/).
 * Plain C11 + pthreads; build: oracle/Makefile.
 */
#define _GNU_SOURCE
#include "kr_oracle.h"

#include <limits.h>
#include <pthread.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#define KR_ID_EMPTY 1u /* interner convention: id 0 = absent, id 1 = "" (include/kr_engine.h) */

/* ------------------------------------------------------------------ SHA-1 (FIPS 180-4) + base32hex (RFC 4648 §7)
 * utils/util.go:634 sha1.Sum, :637 base32.HexEncoding.EncodeToString */

static inline uint32_t rol32(uint32_t x, int n) { return (x << n) | (x >> (32 - n)); }

static void __attribute__((unused)) sha1_block(uint32_t h[5], const uint8_t *p) {
  uint32_t w[80];
  for (int i = 0; i < 16; i++)
    w[i] = ((uint32_t)p[4 * i] << 24) | ((uint32_t)p[4 * i + 1] << 16) | ((uint32_t)p[4 * i + 2] << 8) | p[4 * i + 3];
  for (int i = 16; i < 80; i++) w[i] = rol32(w[i - 3] ^ w[i - 8] ^ w[i - 14] ^ w[i - 16], 1);
  uint32_t a = h[0], b = h[1], c = h[2], d = h[3], e = h[4];
  for (int i = 0; i < 80; i++) {
    uint32_t f, k;
    if (i < 20) { f = (b & c) | (~b & d); k = 0x5A827999u; }
    else if (i < 40) { f = b ^ c ^ d; k = 0x6ED9EBA1u; }
    else if (i < 60) { f = (b & c) | (b & d) | (c & d); k = 0x8F1BBCDCu; }
    else { f = b ^ c ^ d; k = 0xCA62C1D6u; }
    uint32_t t = rol32(a, 5) + f + e + k + w[i];
    e = d; d = c; c = rol32(b, 30); b = a; a = t;
  }
  h[0] += a; h[1] += b; h[2] += c; h[3] += d; h[4] += e;
}

#if defined(__SHA__) && defined(__SSE4_1__)
/* SHA-NI block function (only in the -march=native build bench.py makes for the CPU arm on a host that has the extension):
 * Go's crypto/sha1 uses the same instructions on amd64, so the timed CPU baseline is not handicapped by a portable-C SHA-1.
 * Same FIPS 180-4 compression function as sha1_block; tests/test_oracle_units.py checks both against hashlib. */
#include <immintrin.h>
static void sha1_blocks_ni(uint32_t h[5], const uint8_t *p, uint64_t nblk) {
  const __m128i flip = _mm_set_epi64x(0x0001020304050607ULL, 0x08090a0b0c0d0e0fULL);
  __m128i abcd = _mm_shuffle_epi32(_mm_loadu_si128((const __m128i *)h), 0x1B);
  __m128i e0 = _mm_set_epi32((int)h[4], 0, 0, 0), e1;
  while (nblk--) {
    const __m128i abcd_save = abcd, e_save = e0;
    __m128i m0 = _mm_shuffle_epi8(_mm_loadu_si128((const __m128i *)(p + 0)), flip);
    __m128i m1 = _mm_shuffle_epi8(_mm_loadu_si128((const __m128i *)(p + 16)), flip);
    __m128i m2 = _mm_shuffle_epi8(_mm_loadu_si128((const __m128i *)(p + 32)), flip);
    __m128i m3 = _mm_shuffle_epi8(_mm_loadu_si128((const __m128i *)(p + 48)), flip);
    /* rounds 0-3 */
    e0 = _mm_add_epi32(e0, m0); e1 = abcd; abcd = _mm_sha1rnds4_epu32(abcd, e0, 0);
    /* 4-7 */
    e1 = _mm_sha1nexte_epu32(e1, m1); e0 = abcd; abcd = _mm_sha1rnds4_epu32(abcd, e1, 0); m0 = _mm_sha1msg1_epu32(m0, m1);
    /* 8-11 */
    e0 = _mm_sha1nexte_epu32(e0, m2); e1 = abcd; abcd = _mm_sha1rnds4_epu32(abcd, e0, 0); m1 = _mm_sha1msg1_epu32(m1, m2); m0 = _mm_xor_si128(m0, m2);
    /* 12-15 */
    e1 = _mm_sha1nexte_epu32(e1, m3); e0 = abcd; m0 = _mm_sha1msg2_epu32(m0, m3); abcd = _mm_sha1rnds4_epu32(abcd, e1, 0); m2 = _mm_sha1msg1_epu32(m2, m3); m1 = _mm_xor_si128(m1, m3);
    /* 16-19 */
    e0 = _mm_sha1nexte_epu32(e0, m0); e1 = abcd; m1 = _mm_sha1msg2_epu32(m1, m0); abcd = _mm_sha1rnds4_epu32(abcd, e0, 0); m3 = _mm_sha1msg1_epu32(m3, m0); m2 = _mm_xor_si128(m2, m0);
    /* 20-23 */
    e1 = _mm_sha1nexte_epu32(e1, m1); e0 = abcd; m2 = _mm_sha1msg2_epu32(m2, m1); abcd = _mm_sha1rnds4_epu32(abcd, e1, 1); m0 = _mm_sha1msg1_epu32(m0, m1); m3 = _mm_xor_si128(m3, m1);
    /* 24-27 */
    e0 = _mm_sha1nexte_epu32(e0, m2); e1 = abcd; m3 = _mm_sha1msg2_epu32(m3, m2); abcd = _mm_sha1rnds4_epu32(abcd, e0, 1); m1 = _mm_sha1msg1_epu32(m1, m2); m0 = _mm_xor_si128(m0, m2);
    /* 28-31 */
    e1 = _mm_sha1nexte_epu32(e1, m3); e0 = abcd; m0 = _mm_sha1msg2_epu32(m0, m3); abcd = _mm_sha1rnds4_epu32(abcd, e1, 1); m2 = _mm_sha1msg1_epu32(m2, m3); m1 = _mm_xor_si128(m1, m3);
    /* 32-35 */
    e0 = _mm_sha1nexte_epu32(e0, m0); e1 = abcd; m1 = _mm_sha1msg2_epu32(m1, m0); abcd = _mm_sha1rnds4_epu32(abcd, e0, 1); m3 = _mm_sha1msg1_epu32(m3, m0); m2 = _mm_xor_si128(m2, m0);
    /* 36-39 */
    e1 = _mm_sha1nexte_epu32(e1, m1); e0 = abcd; m2 = _mm_sha1msg2_epu32(m2, m1); abcd = _mm_sha1rnds4_epu32(abcd, e1, 1); m0 = _mm_sha1msg1_epu32(m0, m1); m3 = _mm_xor_si128(m3, m1);
    /* 40-43 */
    e0 = _mm_sha1nexte_epu32(e0, m2); e1 = abcd; m3 = _mm_sha1msg2_epu32(m3, m2); abcd = _mm_sha1rnds4_epu32(abcd, e0, 2); m1 = _mm_sha1msg1_epu32(m1, m2); m0 = _mm_xor_si128(m0, m2);
    /* 44-47 */
    e1 = _mm_sha1nexte_epu32(e1, m3); e0 = abcd; m0 = _mm_sha1msg2_epu32(m0, m3); abcd = _mm_sha1rnds4_epu32(abcd, e1, 2); m2 = _mm_sha1msg1_epu32(m2, m3); m1 = _mm_xor_si128(m1, m3);
    /* 48-51 */
    e0 = _mm_sha1nexte_epu32(e0, m0); e1 = abcd; m1 = _mm_sha1msg2_epu32(m1, m0); abcd = _mm_sha1rnds4_epu32(abcd, e0, 2); m3 = _mm_sha1msg1_epu32(m3, m0); m2 = _mm_xor_si128(m2, m0);
    /* 52-55 */
    e1 = _mm_sha1nexte_epu32(e1, m1); e0 = abcd; m2 = _mm_sha1msg2_epu32(m2, m1); abcd = _mm_sha1rnds4_epu32(abcd, e1, 2); m0 = _mm_sha1msg1_epu32(m0, m1); m3 = _mm_xor_si128(m3, m1);
    /* 56-59 */
    e0 = _mm_sha1nexte_epu32(e0, m2); e1 = abcd; m3 = _mm_sha1msg2_epu32(m3, m2); abcd = _mm_sha1rnds4_epu32(abcd, e0, 2); m1 = _mm_sha1msg1_epu32(m1, m2); m0 = _mm_xor_si128(m0, m2);
    /* 60-63 */
    e1 = _mm_sha1nexte_epu32(e1, m3); e0 = abcd; m0 = _mm_sha1msg2_epu32(m0, m3); abcd = _mm_sha1rnds4_epu32(abcd, e1, 3); m2 = _mm_sha1msg1_epu32(m2, m3); m1 = _mm_xor_si128(m1, m3);
    /* 64-67 */
    e0 = _mm_sha1nexte_epu32(e0, m0); e1 = abcd; m1 = _mm_sha1msg2_epu32(m1, m0); abcd = _mm_sha1rnds4_epu32(abcd, e0, 3); m3 = _mm_sha1msg1_epu32(m3, m0); m2 = _mm_xor_si128(m2, m0);
    /* 68-71 */
    e1 = _mm_sha1nexte_epu32(e1, m1); e0 = abcd; m2 = _mm_sha1msg2_epu32(m2, m1); abcd = _mm_sha1rnds4_epu32(abcd, e1, 3); m3 = _mm_xor_si128(m3, m1);
    /* 72-75 */
    e0 = _mm_sha1nexte_epu32(e0, m2); e1 = abcd; m3 = _mm_sha1msg2_epu32(m3, m2); abcd = _mm_sha1rnds4_epu32(abcd, e0, 3);
    /* 76-79 */
    e1 = _mm_sha1nexte_epu32(e1, m3); e0 = abcd; abcd = _mm_sha1rnds4_epu32(abcd, e1, 3);
    e0 = _mm_sha1nexte_epu32(e0, e_save);
    abcd = _mm_add_epi32(abcd, abcd_save);
    p += 64;
  }
  _mm_storeu_si128((__m128i *)h, _mm_shuffle_epi32(abcd, 0x1B));
  h[4] = (uint32_t)_mm_extract_epi32(e0, 3);
}
#define KR_SHA1_BLOCKS(h, p, n) sha1_blocks_ni(h, p, n)
#else
#define KR_SHA1_BLOCKS(h, p, n) do { for (uint64_t i_ = 0; i_ < (n); i_++) sha1_block(h, (p) + 64 * i_); } while (0)
#endif

void kr_oracle_sha1(const uint8_t *msg, uint64_t len, uint8_t digest[20]) {
  uint32_t h[5] = {0x67452301u, 0xEFCDAB89u, 0x98BADCFEu, 0x10325476u, 0xC3D2E1F0u};
  uint64_t full = len / 64;
  KR_SHA1_BLOCKS(h, msg, full);
  uint8_t tail[128];
  uint64_t rem = len - 64 * full;
  memset(tail, 0, sizeof tail);
  if (rem) memcpy(tail, msg + 64 * full, rem);
  tail[rem] = 0x80;
  int nb = (rem >= 56) ? 2 : 1;
  uint64_t bits = len * 8;
  for (int i = 0; i < 8; i++) tail[64 * nb - 1 - i] = (uint8_t)(bits >> (8 * i));
  KR_SHA1_BLOCKS(h, tail, (uint64_t)nb);
  for (int i = 0; i < 5; i++) {
    digest[4 * i] = (uint8_t)(h[i] >> 24); digest[4 * i + 1] = (uint8_t)(h[i] >> 16);
    digest[4 * i + 2] = (uint8_t)(h[i] >> 8); digest[4 * i + 3] = (uint8_t)h[i];
  }
}

int kr_oracle_sha1_impl(void) {
#if defined(__SHA__) && defined(__SSE4_1__)
  return 1; /* SHA-NI */
#else
  return 0; /* portable C */
#endif
}

void kr_oracle_hash32(const uint8_t *msg, uint64_t len, char out32[32]) {
  static const char alphabet[] = "0123456789ABCDEFGHIJKLMNOPQRSTUV";
  uint8_t d[20];
  kr_oracle_sha1(msg, len, d);
  /* 160 bits = 32 groups of 5 bits, MSB first; no '=' padding is needed */
  for (int i = 0; i < 32; i++) {
    int bit = 5 * i, byte = bit >> 3, off = bit & 7;
    uint32_t v = ((uint32_t)d[byte] << 8) | (byte + 1 < 20 ? d[byte + 1] : 0);
    out32[i] = alphabet[(v >> (11 - off)) & 31];
  }
}

/* ------------------------------------------------------------------ scalar helpers */

/* utils/util.go:386-404.  The multiply is an int32 multiply in Go (wraps). */
int32_t kr_oracle_desired_replicas(int32_t replicas, int32_t min, int32_t max, int32_t num_hosts, uint32_t gflags) {
  int32_t minr = (gflags & KR_GF_MIN_NIL) ? 0 : min;
  int32_t maxr = (gflags & KR_GF_MAX_NIL) ? INT32_MAX : max;
  if (gflags & KR_GF_SUSPEND) return 0;
  int32_t w;
  if ((gflags & KR_GF_REPLICAS_NIL) || replicas < minr) w = minr;
  else if (replicas > maxr) w = maxr;
  else w = replicas;
  return (int32_t)((uint32_t)w * (uint32_t)num_hosts);
}

static inline uint32_t pp_node_type(uint32_t pk) { return (pk >> KR_PP_NODE_TYPE_SHIFT) & 3u; }
static inline uint32_t pp_phase(uint32_t pk) { return (pk >> KR_PP_PHASE_SHIFT) & 7u; }
static inline uint32_t pp_ready(uint32_t pk) { return (pk >> KR_PP_READY_SHIFT) & 3u; }

/* raycluster_controller.go:1181-1231 */
int kr_oracle_should_delete(uint32_t pk) {
  uint32_t ph = pp_phase(pk);
  if (ph == KR_PHASE_FAILED || ph == KR_PHASE_SUCCEEDED) return 1;
  if (ph == KR_PHASE_RUNNING && (pk & KR_PP_RAY_TERMINATED) && (pk & KR_PP_RESTART_NEVER)) return 1;
  return 0;
}

/* ------------------------------------------------------------------ u64 -> u32 open-addressing map */

typedef struct { uint64_t *keys; uint32_t *vals; uint64_t mask; } kmap;
#define KMAP_EMPTY 0xFFFFFFFFFFFFFFFFull

static uint64_t mix64(uint64_t x) {
  x ^= x >> 33; x *= 0xff51afd7ed558ccdull; x ^= x >> 33; x *= 0xc4ceb9fe1a85ec53ull; x ^= x >> 33;
  return x;
}
static int kmap_init(kmap *m, uint64_t n) {
  uint64_t cap = 16;
  while (cap < 2 * n + 2) cap <<= 1;
  m->keys = (uint64_t *)malloc(cap * sizeof(uint64_t));
  m->vals = (uint32_t *)malloc(cap * sizeof(uint32_t));
  if (!m->keys || !m->vals) return -1;
  memset(m->keys, 0xFF, cap * sizeof(uint64_t));
  m->mask = cap - 1;
  return 0;
}
static void kmap_free(kmap *m) { free(m->keys); free(m->vals); m->keys = NULL; m->vals = NULL; }
/* insert if absent (first writer wins => lowest index when inserted in ascending order) */
static void kmap_put_first(kmap *m, uint64_t k, uint32_t v) {
  uint64_t i = mix64(k) & m->mask;
  while (m->keys[i] != KMAP_EMPTY) { if (m->keys[i] == k) return; i = (i + 1) & m->mask; }
  m->keys[i] = k; m->vals[i] = v;
}
static int kmap_get(const kmap *m, uint64_t k, uint32_t *v) {
  uint64_t i = mix64(k) & m->mask;
  while (m->keys[i] != KMAP_EMPTY) { if (m->keys[i] == k) { *v = m->vals[i]; return 1; } i = (i + 1) & m->mask; }
  return 0;
}
static inline uint64_t key2(uint32_t a, uint32_t b) { return ((uint64_t)a << 32) | b; }

/* ------------------------------------------------------------------ shared read-only context */

typedef struct {
  const kr_snapshot_bufs *s;
  const kr_sizes *n;
  const kr_flags *f;
  kr_oracle_out *out;
  int list_mode;
  kmap cluster_map;  /* (ns,name) -> cluster idx */
  kmap podname_map;  /* (ns,name) -> pod idx (lowest) */
  kmap ns_map;       /* ns_id -> dense bucket */
  uint32_t *pod_cluster;   /* [Np] cluster idx or n_clusters (orphan) */
  uint32_t *cl_start;      /* [Nc+2] bucket offsets (bucket Nc = orphans) */
  uint32_t *cl_pods;       /* [Np] pods bucketed by cluster, list order */
  uint32_t *ns_start;      /* [Nns+1] */
  uint32_t *ns_pods;       /* [Np] pods bucketed by namespace, list order */
  int32_t  *pod_head_aux;  /* [Np] head-aux row or -1 */
  int32_t  *wtd;           /* [Nw] pod a workersToDelete name resolves to (same namespace + same name), -1 = NotFound */
  uint8_t  *act;           /* [Np] action by original pod index */
} octx;

/* A "listed" pod: what a cached List hands back (a copy of the object, here of its columns). */
typedef struct {
  uint32_t idx, name_id, group_name_id, packed, replica_name_id;
  int32_t replica_index;
} lpod;

typedef struct { lpod *v; uint32_t n, cap; } lvec;
static void lvec_push(lvec *l, const lpod *p) {
  if (l->n == l->cap) { l->cap = l->cap ? 2 * l->cap : 64; l->v = (lpod *)realloc(l->v, l->cap * sizeof(lpod)); }
  l->v[l->n++] = *p;
}

static inline void load_pod(const kr_snapshot_bufs *s, uint32_t p, lpod *o) {
  o->idx = p; o->name_id = s->p_name_id[p]; o->group_name_id = s->p_group_name_id[p];
  o->packed = s->p_packed[p]; o->replica_name_id = s->p_replica_name_id[p]; o->replica_index = s->p_replica_index[p];
}

/* selector kinds: common/association.go:83-130 */
enum { SEL_ALL = 0, SEL_HEAD = 1, SEL_GROUP = 2 };

/* r.List(ctx, &pods, InNamespace(ns), MatchingLabels{ray.io/cluster: name [, node-type: head | group: g]}) */
static void list_pods(const octx *x, uint32_t c, int sel, uint32_t group_name_id, lvec *out) {
  const kr_snapshot_bufs *s = x->s;
  out->n = 0;
  lpod lp;
  if (x->list_mode == KR_ORACLE_INDEXED) {
    for (uint32_t i = x->cl_start[c]; i < x->cl_start[c + 1]; i++) {
      uint32_t p = x->cl_pods[i];
      if (sel == SEL_HEAD && pp_node_type(s->p_packed[p]) != KR_NT_HEAD) continue;
      if (sel == SEL_GROUP && (group_name_id == 0 || s->p_group_name_id[p] != group_name_id)) continue;
      load_pod(s, p, &lp); lvec_push(out, &lp);
    }
    return;
  }
  /* NS_SCAN: walk every cached pod of the namespace and test the label selector (SURVEY §3.2(a)) */
  uint32_t b;
  if (!kmap_get(&x->ns_map, s->c_ns_id[c], &b)) return;
  uint32_t cname = s->c_name_id[c];
  for (uint32_t i = x->ns_start[b]; i < x->ns_start[b + 1]; i++) {
    uint32_t p = x->ns_pods[i];
    if (cname == 0 || s->p_cluster_name_id[p] != cname) continue;
    if (sel == SEL_HEAD && pp_node_type(s->p_packed[p]) != KR_NT_HEAD) continue;
    if (sel == SEL_GROUP && (group_name_id == 0 || s->p_group_name_id[p] != group_name_id)) continue;
    load_pod(s, p, &lp); lvec_push(out, &lp);
  }
}

/* per-thread scratch */
typedef struct {
  lvec heads, group, all, tmp;
  uint8_t *deleted;      /* per list position */
  uint32_t deleted_cap;
  /* multi-host */
  uint32_t *rep_key, *rep_cnt, *rep_first, *rep_flags, *rep_slot_of_pos;
  uint32_t rep_cap;
  uint8_t *bitmap; uint64_t bitmap_cap;
} oscratch;

static void scratch_free(oscratch *t) {
  free(t->heads.v); free(t->group.v); free(t->all.v); free(t->tmp.v); free(t->deleted);
  free(t->rep_key); free(t->rep_cnt); free(t->rep_first); free(t->rep_flags); free(t->rep_slot_of_pos); free(t->bitmap);
}

/* Lowest `want` non-negative integers not present among idx[0..n) (only entries flagged valid).
 * raycluster_controller.go:854-881 and :1066-1094. */
static void alloc_lowest_free(oscratch *t, const int32_t *idx, const uint8_t *valid, uint32_t n, uint32_t want, int32_t *dst) {
  uint64_t bound = (uint64_t)n + want; /* the `want` lowest free indices all lie below n+want */
  uint64_t bytes = (bound + 7) / 8;
  if (bytes > t->bitmap_cap) { t->bitmap_cap = bytes * 2; t->bitmap = (uint8_t *)realloc(t->bitmap, t->bitmap_cap); }
  memset(t->bitmap, 0, bytes);
  for (uint32_t i = 0; i < n; i++)
    if (valid[i] && idx[i] >= 0 && (uint64_t)idx[i] < bound) t->bitmap[idx[i] >> 3] |= (uint8_t)(1u << (idx[i] & 7));
  uint32_t got = 0;
  for (uint64_t k = 0; k < bound && got < want; k++)
    if (!(t->bitmap[k >> 3] & (1u << (k & 7)))) dst[got++] = (int32_t)k;
}

/* ------------------------------------------------------------------ multi-host group (raycluster_controller.go:963-1125)
 * Deterministic choices where the reference iterates a Go map (SURVEY Appendix A.5): replicas are ordered by
 * first appearance in list order. Returns err_kind (0 = nil) and fills the group result. */
#define REP_DELETED 1u
#define REP_WTD 2u

static int reconcile_multihost(const octx *x, oscratch *t, uint32_t c, uint32_t g, int32_t expected,
                               kr_group_result *gr, int32_t *err_arg, int32_t *create_tmp, uint32_t *n_create_out) {
  const kr_snapshot_bufs *s = x->s;
  lvec *L = &t->group;
  uint32_t n = L->n;
  int32_t H = s->g_num_hosts[g];
  if (n + 1 > t->rep_cap) {
    t->rep_cap = 2 * (n + 1);
    t->rep_key = (uint32_t *)realloc(t->rep_key, t->rep_cap * 4); t->rep_cnt = (uint32_t *)realloc(t->rep_cnt, t->rep_cap * 4);
    t->rep_first = (uint32_t *)realloc(t->rep_first, t->rep_cap * 4); t->rep_flags = (uint32_t *)realloc(t->rep_flags, t->rep_cap * 4);
    t->rep_slot_of_pos = (uint32_t *)realloc(t->rep_slot_of_pos, t->rep_cap * 4);
  }
  /* 1. replicaMap: group by ray.io/worker-group-replica-name (:967-972); slots in first-appearance order */
  uint32_t R = 0;
  for (uint32_t i = 0; i < n; i++) {
    uint32_t key = L->v[i].replica_name_id;
    t->rep_slot_of_pos[i] = UINT32_MAX;
    if (key == 0) continue; /* label absent: pod is in no replica */
    uint32_t r;
    for (r = 0; r < R; r++) if (t->rep_key[r] == key) break;
    if (r == R) { t->rep_key[R] = key; t->rep_cnt[R] = 0; t->rep_first[R] = i; t->rep_flags[R] = 0; R++; }
    t->rep_cnt[r]++;
    t->rep_slot_of_pos[i] = r;
  }
  /* 2. incomplete replica groups (:975-984) */
  for (uint32_t r = 0; r < R; r++) {
    if ((int64_t)t->rep_cnt[r] < (int64_t)H) {
      for (uint32_t i = 0; i < n; i++)
        if (t->rep_slot_of_pos[i] == r) x->act[L->v[i].idx] = KR_ACT_DELETE_MH_INCOMPLETE;
      gr->flags |= KR_GR_ABORTED;
      *err_arg = (int32_t)t->rep_cnt[r];
      return KR_ERR_MH_INCOMPLETE;
    }
  }
  /* 3. unhealthy replica groups (:987-1007) */
  uint32_t n_unhealthy = 0;
  for (uint32_t i = 0; i < n; i++) {
    if (x->act[L->v[i].idx] != KR_ACT_KEEP) continue; /* alreadyDeleted */
    if (!kr_oracle_should_delete(L->v[i].packed)) continue;
    uint32_t key = L->v[i].replica_name_id ? L->v[i].replica_name_id : KR_ID_EMPTY;
    uint32_t r;
    for (r = 0; r < R; r++) if (t->rep_key[r] == key) break;
    if (r == R) continue; /* replicaMap[replicaName] !ok */
    t->rep_flags[r] |= REP_DELETED;
    for (uint32_t k = 0; k < n; k++)
      if (t->rep_slot_of_pos[k] == r && x->act[L->v[k].idx] == KR_ACT_KEEP) { x->act[L->v[k].idx] = KR_ACT_DELETE_MH_UNHEALTHY; n_unhealthy++; }
  }
  gr->n_unhealthy = (int32_t)n_unhealthy;
  /* 4. explicit deletions from the autoscaler (:1010-1038) */
  uint32_t wc = s->g_wtd_cnt[g];
  if (wc > 0) {
    uint32_t n_del = 0;
    for (uint32_t w = 0; w < wc; w++) {
      uint32_t name = s->w_name_id[s->g_wtd_off[g] + w];
      for (uint32_t i = 0; i < n; i++) {
        if (L->v[i].name_id != name) continue;
        uint32_t key = L->v[i].replica_name_id ? L->v[i].replica_name_id : KR_ID_EMPTY;
        for (uint32_t r = 0; r < R; r++) if (t->rep_key[r] == key) t->rep_flags[r] |= REP_WTD;
        break;
      }
    }
    for (uint32_t i = 0; i < n; i++) {
      uint32_t r = t->rep_slot_of_pos[i];
      if (r != UINT32_MAX && (t->rep_flags[r] & REP_WTD)) {
        n_del++;
        if (x->act[L->v[i].idx] == KR_ACT_KEEP) x->act[L->v[i].idx] = KR_ACT_DELETE_MH_WTD;
      }
    }
    gr->flags |= KR_GR_WTD_EXECUTED;
    if (n_del > 0) { gr->flags |= KR_GR_ABORTED; *err_arg = (int32_t)n_del; return KR_ERR_MH_WTD; }
  }
  /* 5. diff by replica (:1042-1064) */
  int32_t running = 0;
  for (uint32_t r = 0; r < R; r++) if (!(t->rep_flags[r] & REP_DELETED)) running++;
  gr->n_running = running;
  if (H == 0 || expected % H != 0) { gr->flags |= KR_GR_ABORTED; *err_arg = expected; return KR_ERR_MH_NOT_MULTIPLE; }
  int32_t to_create = expected / H - running;
  gr->diff = to_create;
  if (to_create > 0) {
    /* in-use indices: label of the first pod of every valid replica (:1067-1077) */
    int32_t *idx = (int32_t *)malloc((R + 1) * sizeof(int32_t));
    uint8_t *valid = (uint8_t *)malloc(R + 1);
    uint32_t m = 0;
    for (uint32_t r = 0; r < R; r++) {
      if (t->rep_flags[r] & REP_DELETED) continue;
      const lpod *p = &L->v[t->rep_first[r]];
      idx[m] = p->replica_index; valid[m] = (p->packed & KR_PP_HAS_REPLICA_IDX) ? 1 : 0; m++;
    }
    alloc_lowest_free(t, idx, valid, m, (uint32_t)to_create, create_tmp);
    free(idx); free(valid);
    *n_create_out = (uint32_t)to_create;
  } else if (to_create < 0) {
    int autoscaling = (s->c_flags[c] & KR_CF_AUTOSCALING) != 0;
    if (!autoscaling || x->f->env_random_pod_delete) {
      int32_t remove = -to_create, removed = 0;
      for (uint32_t r = 0; r < R && removed < remove; r++) {
        if (t->rep_flags[r] & REP_DELETED) continue;
        for (uint32_t i = 0; i < n; i++)
          if (t->rep_slot_of_pos[i] == r) x->act[L->v[i].idx] = KR_ACT_DELETE_MH_SCALE_DOWN;
        removed++;
      }
    } else {
      gr->flags |= KR_GR_RANDOM_DELETE_OFF;
    }
  }
  return KR_ERR_NONE;
}

/* ------------------------------------------------------------------ reconcilePods (raycluster_controller.go:619-935) */

typedef struct { int32_t *v; uint32_t n, cap; } ivec;
/* Room for `need` entries.  The sum is taken in 64 bits: a RayCluster's groups may together ask for more than 2^31 pods, and a
 * 32-bit size would wrap to a short buffer.  A stream the 32-bit counts cannot describe (or memory cannot hold) stops the process. */
static void ivec_reserve(ivec *v, uint64_t need) {
  if (need <= v->cap) return;
  const uint64_t cap = need * 2 <= UINT32_MAX ? need * 2 : need;
  int32_t *p = cap <= UINT32_MAX ? (int32_t *)realloc(v->v, (size_t)cap * sizeof(int32_t)) : NULL;
  if (!p) { fprintf(stderr, "kr_oracle: a create stream of %llu entries\n", (unsigned long long)need); abort(); }
  v->v = p; v->cap = (uint32_t)cap;
}

static void reconcile_pods(const octx *x, oscratch *t, uint32_t c, const char *hash32, kr_cluster_result *cr,
                           ivec *creates /* (group, n, indices...) stream */) {
  const kr_snapshot_bufs *s = x->s;
  const kr_flags *f = x->f;
  uint32_t cf = s->c_flags[c];
  uint32_t G = s->c_group_cnt[c], g0 = s->c_group_off[c];
  uint8_t suspend_status = s->c_suspend_status[c];
  int gate = f->gate_status_conditions != 0;

  cr->stop_after_group = -1;

  /* :629-644 suspending => delete all pods */
  if (suspend_status == KR_SUSPEND_SUSPENDING || (!gate && (cf & KR_CF_SUSPEND))) {
    list_pods(x, c, SEL_ALL, 0, &t->all);
    for (uint32_t i = 0; i < t->all.n; i++) x->act[t->all.v[i].idx] = KR_ACT_DELETE_ALL_SUSPEND;
    cr->path = KR_PATH_SUSPENDING_DELETE_ALL;
    return;
  }
  /* :646-654 */
  if (gate && (suspend_status == KR_SUSPEND_SUSPENDED || (cf & KR_CF_SUSPEND))) {
    cr->path = KR_PATH_SUSPENDED_NOOP;
    return;
  }
  /* :657 shouldRecreatePodsForUpgrade (:1132-1171) */
  if (cf & KR_CF_UPGRADE_RECREATE) {
    list_pods(x, c, SEL_HEAD, 0, &t->heads);
    if (t->heads.n > 0) {
      int32_t aux = x->pod_head_aux[t->heads.v[0].idx];
      uint8_t ver = aux >= 0 ? s->h_version_state[aux] : KR_VER_EMPTY;
      uint8_t ast = aux >= 0 ? s->h_annot_state[aux] : KR_ANNOT_EMPTY;
      if (ver == KR_VER_DIFFERENT) {
        cr->head_update_annotations = 1; /* :1155-1162, then continue normally */
      } else {
        int differs = 0;
        if (ast == KR_ANNOT_OTHER) differs = 1;
        else if (ast == KR_ANNOT_HASH32) differs = f->skip_hash ? 0 : (memcmp(s->h_annot_hash + 32 * (size_t)aux, hash32, 32) != 0);
        if (differs) { /* :1165-1168 => :658-669 */
          list_pods(x, c, SEL_ALL, 0, &t->all);
          for (uint32_t i = 0; i < t->all.n; i++) x->act[t->all.v[i].idx] = KR_ACT_DELETE_ALL_RECREATE;
          cr->path = KR_PATH_RECREATE_DELETE_ALL;
          return;
        }
      }
    }
  }
  cr->path = KR_PATH_NORMAL;

  /* :673-748 head pod */
  list_pods(x, c, SEL_HEAD, 0, &t->heads);
  if (!(cf & KR_CF_HEAD_EXPECT_OK)) {
    cr->head_action = KR_HEAD_EXPECT_PENDING;
  } else if (t->heads.n == 1) {
    if (kr_oracle_should_delete(t->heads.v[0].packed)) {
      x->act[t->heads.v[0].idx] = KR_ACT_DELETE_HEAD;
      cr->head_action = KR_HEAD_DELETE;
      cr->err_kind = KR_ERR_HEAD_DELETED;
      return;
    }
  } else if (t->heads.n == 0) {
    int provisioned = s->c_old_cond_status[5 * (size_t)c + KR_COND_PROVISIONED] == KR_COND_TRUE;
    if (provisioned && (cf & KR_CF_SKIP_HEAD_RESTART)) { cr->head_action = KR_HEAD_SKIP_RESTART; return; }
    cr->head_action = KR_HEAD_CREATE;
  } else {
    cr->head_action = KR_HEAD_MULTIPLE;
    cr->err_kind = KR_ERR_MULTIPLE_HEADS;
    cr->err_arg = (int32_t)t->heads.n;
    return;
  }

  /* :751-933 worker groups in spec order */
  for (uint32_t gi = 0; gi < G; gi++) {
    uint32_t g = g0 + gi;
    kr_group_result *gr = &x->out->groups[g];
    uint32_t gf = s->g_flags[g];
    cr->stop_after_group = (int32_t)gi;
    gr->flags = KR_GR_PROCESSED;
    if (!(gf & KR_GF_EXPECT_OK)) { gr->flags |= KR_GR_EXPECT_PENDING; continue; }
    int32_t expected = kr_oracle_desired_replicas(s->g_replicas[g], s->g_min[g], s->g_max[g], s->g_num_hosts[g], gf);
    gr->expected = expected;
    list_pods(x, c, SEL_GROUP, s->g_name_id[g], &t->group);
    lvec *L = &t->group;
    gr->n_list = (int32_t)L->n;
    if (gf & KR_GF_SUSPEND) { /* :766-775 */
      for (uint32_t i = 0; i < L->n; i++) x->act[L->v[i].idx] = KR_ACT_DELETE_GROUP_SUSPEND;
      gr->flags |= KR_GR_SUSPENDED;
      continue;
    }
    if (s->g_num_hosts[g] > 1 && f->gate_multihost_indexing) { /* :777-784 */
      gr->flags |= KR_GR_MULTIHOST;
      uint32_t want = 0;
      uint32_t need = expected > 0 ? (uint32_t)expected : 0;
      int32_t *tmp = (int32_t *)malloc(((size_t)need + 1) * sizeof(int32_t));
      int32_t earg = 0;
      int ek = reconcile_multihost(x, t, c, g, expected, gr, &earg, tmp, &want);
      if (ek == KR_ERR_NONE && want) {
        gr->n_create = want;
        ivec_reserve(creates, (uint64_t)creates->n + 2 + want);
        creates->v[creates->n++] = (int32_t)g; creates->v[creates->n++] = (int32_t)want;
        memcpy(creates->v + creates->n, tmp, want * sizeof(int32_t)); creates->n += want;
      }
      free(tmp);
      if (ek != KR_ERR_NONE) { cr->err_kind = (uint8_t)ek; cr->err_arg = earg; return; }
      continue;
    }
    /* :786-812 unhealthy workers, list order */
    if (L->n > t->deleted_cap) { t->deleted_cap = 2 * L->n; t->deleted = (uint8_t *)realloc(t->deleted, t->deleted_cap); }
    memset(t->deleted, 0, L->n);
    int32_t n_unhealthy = 0;
    for (uint32_t i = 0; i < L->n; i++) {
      if (kr_oracle_should_delete(L->v[i].packed)) { n_unhealthy++; t->deleted[i] = 1; x->act[L->v[i].idx] = KR_ACT_DELETE_UNHEALTHY; }
    }
    gr->n_unhealthy = n_unhealthy;
    if (n_unhealthy > 0) {
      gr->flags |= KR_GR_ABORTED;
      cr->err_kind = KR_ERR_UNHEALTHY_WORKERS; cr->err_arg = n_unhealthy;
      return;
    }
    /* :814-835 WorkersToDelete: r.Delete(ns, name); success => deletedWorkers[name] */
    gr->flags |= KR_GR_WTD_EXECUTED;
    for (uint32_t w = 0; w < s->g_wtd_cnt[g]; w++) {
      int32_t j = x->wtd[s->g_wtd_off[g] + w]; /* resolved up front: same namespace + same name */
      if (j < 0) continue;                                    /* NotFound: tolerated (:823-828) */
      uint32_t name = s->p_name_id[j];
      for (uint32_t i = 0; i < L->n; i++)
        if (L->v[i].name_id == name) { t->deleted[i] = 1; x->act[L->v[i].idx] = KR_ACT_DELETE_WTD; }
    }
    /* :837-849 runningPods, diff */
    int32_t running = 0;
    for (uint32_t i = 0; i < L->n; i++) if (!t->deleted[i]) running++;
    gr->n_running = running;
    /* Go's int32 arithmetic wraps (:836): an expected count near -2^31 turns into billions of pods to create.  The subtraction is done
     * in uint32_t so that the wrap is defined here too; such a stream is a capacity error, and ivec_reserve stops the process if it
     * cannot even be counted (tests/fuzz_objects.py keeps |expected| <= 300 for that reason). */
    int32_t diff = (int32_t)((uint32_t)expected - (uint32_t)running);
    gr->diff = diff;
    if (diff > 0) { /* :865-890 */
      uint32_t want = (uint32_t)diff;
      gr->n_create = want;
      ivec_reserve(creates, (uint64_t)creates->n + 2 + want);
      creates->v[creates->n++] = (int32_t)g; creates->v[creates->n++] = (int32_t)want;
      int32_t *dst = creates->v + creates->n;
      if (f->gate_multihost_indexing) {
        int32_t *idx = (int32_t *)malloc(((size_t)running + 1) * sizeof(int32_t));
        uint8_t *valid = (uint8_t *)malloc((size_t)running + 1);
        uint32_t m = 0;
        for (uint32_t i = 0; i < L->n; i++) {
          if (t->deleted[i]) continue;
          idx[m] = L->v[i].replica_index; valid[m] = (L->v[i].packed & KR_PP_HAS_REPLICA_IDX) ? 1 : 0; m++;
        }
        alloc_lowest_free(t, idx, valid, m, want, dst);
        free(idx); free(valid);
      } else {
        for (uint32_t k = 0; k < want; k++) dst[k] = -1; /* createWorkerPod without index (:884-889) */
      }
      creates->n += want;
    } else if (diff < 0) { /* :894-932 */
      int autoscaling = (cf & KR_CF_AUTOSCALING) != 0;
      if (!autoscaling || f->env_random_pod_delete) {
        int64_t remove = -(int64_t)diff;
        int64_t done = 0;
        for (uint32_t i = 0; i < L->n && done < remove; i++) {
          if (t->deleted[i]) continue;
          x->act[L->v[i].idx] = KR_ACT_DELETE_RANDOM; done++;
        }
        if (done < remove) { /* expected < 0: Go would index past runningPods (:917) */
          gr->flags |= KR_GR_ABORTED;
          cr->err_kind = KR_ERR_NEGATIVE_EXPECTED; cr->err_arg = expected;
          return;
        }
      } else {
        gr->flags |= KR_GR_RANDOM_DELETE_OFF;
      }
    }
  }
  cr->stop_after_group = (int32_t)G;
}

/* ------------------------------------------------------------------ calculateStatus (raycluster_controller.go:1552-1719) */

static void calculate_status(const octx *x, oscratch *t, uint32_t c, kr_cluster_result *cr) {
  const kr_snapshot_bufs *s = x->s;
  const kr_flags *f = x->f;
  uint32_t cf = s->c_flags[c];
  int gate = f->gate_status_conditions != 0;
  int reconcile_err = cr->err_kind != KR_ERR_NONE;
  uint8_t ek = s->c_ext_err_kind[c];

  uint8_t cst[KR_NUM_CONDS], cvr[KR_NUM_CONDS];
  for (int k = 0; k < KR_NUM_CONDS; k++) { cst[k] = s->c_old_cond_status[5 * (size_t)c + k]; cvr[k] = s->c_old_cond_variant[5 * (size_t)c + k]; }
  uint32_t hpr_reason = s->c_old_cond_reason_id[c], hpr_msg = s->c_old_cond_msg_id[2 * (size_t)c];
  uint32_t rf_msg = s->c_old_cond_msg_id[2 * (size_t)c + 1];

  /* :1563-1577 ReplicaFailure */
  if (gate) {
    if (reconcile_err) {
      if (ek >= KR_EXT_ERR_FAILED_DELETE_ALL_PODS && ek <= KR_EXT_ERR_FAILED_CREATE_WORKER_POD) {
        cst[KR_COND_REPLICA_FAILURE] = KR_COND_TRUE; cvr[KR_COND_REPLICA_FAILURE] = ek; rf_msg = s->c_ext_err_msg_id[c];
      }
    } else {
      cst[KR_COND_REPLICA_FAILURE] = KR_COND_ABSENT; cvr[KR_COND_REPLICA_FAILURE] = KR_CV_NONE; rf_msg = 0;
    }
  }

  /* :1582-1591 */
  list_pods(x, c, SEL_ALL, 0, &t->all);
  lvec *P = &t->all;
  int32_t ready = 0, available = 0;
  int all_running = P->n > 0; /* utils/util.go:584-603 */
  uint32_t n_heads = 0; int32_t head_pos = -1;
  for (uint32_t i = 0; i < P->n; i++) {
    uint32_t pk = P->v[i].packed;
    uint32_t nt = pp_node_type(pk), ph = pp_phase(pk), rd = pp_ready(pk);
    if (nt == KR_NT_WORKER) { /* utils/util.go:446-474 */
      if (ph == KR_PHASE_RUNNING) { available++; if (rd == KR_COND_TRUE) ready++; }
    }
    if (ph != KR_PHASE_RUNNING || rd == KR_COND_FALSE || rd == KR_COND_UNKNOWN) all_running = 0;
    if (nt == KR_NT_HEAD) { if (n_heads == 0) head_pos = (int32_t)i; n_heads++; }
  }
  int32_t desired = 0, minr = 0; int64_t maxr = 0;
  uint32_t G = s->c_group_cnt[c], g0 = s->c_group_off[c];
  for (uint32_t gi = 0; gi < G; gi++) { /* utils/util.go:407-442 */
    uint32_t g = g0 + gi, gf = s->g_flags[g];
    desired = (int32_t)((uint32_t)desired + (uint32_t)kr_oracle_desired_replicas(s->g_replicas[g], s->g_min[g], s->g_max[g], s->g_num_hosts[g], gf));
    if (gf & KR_GF_SUSPEND) continue;
    int32_t mn = (gf & KR_GF_MIN_NIL) ? 0 : s->g_min[g];
    int32_t mx = (gf & KR_GF_MAX_NIL) ? INT32_MAX : s->g_max[g];
    minr = (int32_t)((uint32_t)minr + (uint32_t)mn * (uint32_t)s->g_num_hosts[g]);
    maxr += (int64_t)mx * (int64_t)s->g_num_hosts[g];
  }
  int32_t maxc = maxr > INT32_MAX ? INT32_MAX : (maxr < INT32_MIN ? INT32_MIN : (int32_t)maxr); /* utils/util.go:284-292 */

  cr->n_pods = (int32_t)P->n;
  cr->n_heads = (int32_t)n_heads;
  cr->head_pod_idx = head_pos >= 0 ? (int32_t)P->v[head_pos].idx : -1;

  /* errors that make calculateStatus return (nil, err): :1608-1611, :1785-1806 */
  uint8_t serr = KR_SERR_NONE;
  if (n_heads > 1) serr = KR_SERR_MULTIPLE_HEADS;
  else if (s->c_svc_count[c] == 0) serr = KR_SERR_NO_HEAD_SERVICE;
  else if (s->c_svc_count[c] > 1) serr = KR_SERR_MULTIPLE_HEAD_SERVICES;
  else if (s->c_svc_ip_kind[c] == KR_SVCIP_EMPTY) serr = KR_SERR_EMPTY_SERVICE_IP;
  if (x->list_mode == KR_ORACLE_NS_SCAN) { /* the reference issues these Lists (association.go:184 via :1608, :1786) */
    list_pods(x, c, SEL_HEAD, 0, &t->tmp);
    list_pods(x, c, SEL_HEAD, 0, &t->tmp);
  }
  cr->status_err = serr;
  if (serr != KR_SERR_NONE) return; /* all status fields stay zero */

  uint8_t old_state = s->c_old_state[c], new_state = old_state;
  int reason_cleared = 0;
  /* :1599-1604 */
  if (!reconcile_err && (int64_t)P->n == (int64_t)desired + 1 && all_running) { new_state = KR_STATE_READY; reason_cleared = 1; }

  uint32_t head_pod_ip = 0, head_pod_name = 0;
  if (n_heads == 1) {
    int32_t aux = x->pod_head_aux[P->v[head_pos].idx];
    head_pod_ip = aux >= 0 ? s->h_pod_ip_id[aux] : 0;
    head_pod_name = P->v[head_pos].name_id;
  }
  if (gate) {
    /* :1608-1623 HeadPodReady */
    if (n_heads == 0) {
      cst[KR_COND_HEAD_POD_READY] = KR_COND_FALSE; cvr[KR_COND_HEAD_POD_READY] = KR_CV_HEAD_NOT_FOUND;
      hpr_reason = f->id_head_not_found_reason; hpr_msg = f->id_head_not_found_msg;
    } else {
      int32_t aux = x->pod_head_aux[P->v[head_pos].idx];
      cst[KR_COND_HEAD_POD_READY] = aux >= 0 ? s->h_ready_status[aux] : KR_COND_FALSE;
      cvr[KR_COND_HEAD_POD_READY] = KR_CV_HEAD_FROM_POD;
      hpr_reason = aux >= 0 ? s->h_ready_reason_id[aux] : 0; hpr_msg = aux >= 0 ? s->h_ready_msg_id[aux] : 0;
    }
    uint8_t ss = s->c_suspend_status[c];
    /* :1625-1644 */
    if (cst[KR_COND_PROVISIONED] != KR_COND_TRUE && ss != KR_SUSPEND_SUSPENDED) {
      if (all_running) { cst[KR_COND_PROVISIONED] = KR_COND_TRUE; cvr[KR_COND_PROVISIONED] = KR_CV_PROV_ALL_READY; }
      else { cst[KR_COND_PROVISIONED] = KR_COND_FALSE; cvr[KR_COND_PROVISIONED] = KR_CV_PROV_PROVISIONING; }
    }
    /* :1646-1693 */
    if (ss == KR_SUSPEND_SUSPENDING) {
      if (P->n == 0) {
        cst[KR_COND_PROVISIONED] = KR_COND_FALSE; cvr[KR_COND_PROVISIONED] = KR_CV_PROV_SUSPENDED;
        cst[KR_COND_SUSPENDING] = KR_COND_FALSE; cvr[KR_COND_SUSPENDING] = KR_CV_CANONICAL;
        cst[KR_COND_SUSPENDED] = KR_COND_TRUE; cvr[KR_COND_SUSPENDED] = KR_CV_CANONICAL;
      }
    } else if (ss == KR_SUSPEND_SUSPENDED) {
      if (cf & KR_CF_SUSPEND_SET_FALSE) { cst[KR_COND_SUSPENDED] = KR_COND_FALSE; cvr[KR_COND_SUSPENDED] = KR_CV_CANONICAL; }
    } else {
      cst[KR_COND_SUSPENDED] = KR_COND_FALSE; cvr[KR_COND_SUSPENDED] = KR_CV_CANONICAL;
      cst[KR_COND_SUSPENDING] = (cf & KR_CF_SUSPEND) ? KR_COND_TRUE : KR_COND_FALSE; cvr[KR_COND_SUSPENDING] = KR_CV_CANONICAL;
    }
  }
  /* :1696-1698 */
  if ((cf & KR_CF_SUSPEND) && P->n == 0) new_state = KR_STATE_SUSPENDED;

  /* :1785-1806 head info, :1721-1745 service ip */
  uint32_t svc_ip = s->c_svc_ip_id[c];
  if (s->c_svc_ip_kind[c] == KR_SVCIP_NONE) svc_ip = (n_heads == 1) ? head_pod_ip : 0;
  uint32_t head_ids[4] = {head_pod_ip, svc_ip, head_pod_name, s->c_svc_name_id[c]};

  cr->new_state = new_state;
  cr->state_changed = new_state != old_state; /* :1711-1716 */
  cr->status_flags = (reason_cleared ? KR_SF_READY_BRANCH : 0u) | (all_running ? KR_SF_ALL_PODS_RUNNING : 0u);
  cr->counts[0] = ready; cr->counts[1] = available; cr->counts[2] = desired; cr->counts[3] = minr; cr->counts[4] = maxc;
  for (int k = 0; k < KR_NUM_CONDS; k++) { cr->cond_status[k] = cst[k]; cr->cond_variant[k] = cvr[k]; }
  cr->head_ready_reason_id = hpr_reason; cr->head_ready_msg_id = hpr_msg;
  for (int k = 0; k < 4; k++) cr->head_ids[k] = head_ids[k];

  /* utils/consistency.go:16-34 */
  int inc = 0;
  if (new_state != old_state) inc = 1;
  if (reason_cleared && (cf & KR_CF_OLD_REASON_NONEMPTY)) inc = 1;
  for (int k = 0; k < 5; k++) if (s->c_old_counts[5 * (size_t)c + k] != cr->counts[k]) inc = 1;
  if (cf & KR_CF_ENDPOINTS_CHANGED) inc = 1;
  for (int k = 0; k < 4; k++) if (s->c_old_head_ids[4 * (size_t)c + k] != head_ids[k]) inc = 1;
  for (int k = 0; k < KR_NUM_CONDS; k++) {
    uint8_t os = s->c_old_cond_status[5 * (size_t)c + k], ov = s->c_old_cond_variant[5 * (size_t)c + k];
    if (os != cst[k]) { inc = 1; continue; }
    if (cst[k] == KR_COND_ABSENT) continue;
    if (k == KR_COND_HEAD_POD_READY) {
      /* reason/message compared as interned strings */
      if (s->c_old_cond_reason_id[c] != hpr_reason || s->c_old_cond_msg_id[2 * (size_t)c] != hpr_msg) inc = 1;
    } else if (k == KR_COND_REPLICA_FAILURE) {
      if (ov != cvr[k] || s->c_old_cond_msg_id[2 * (size_t)c + 1] != rf_msg) inc = 1;
    } else {
      if (ov != cvr[k]) inc = 1;
    }
  }
  cr->needs_status_write = (uint8_t)inc;
}

/* ------------------------------------------------------------------ driver */

typedef struct {
  octx *x;
  uint32_t c0, c1;
  int reps;
  ivec creates;
  int rc;
} worker_arg;

static void reconcile_cluster(octx *x, oscratch *t, uint32_t c, ivec *creates) {
  const kr_snapshot_bufs *s = x->s;
  kr_cluster_result *cr = &x->out->clusters[c];
  memset(cr, 0, sizeof *cr);
  cr->head_pod_idx = -1;
  cr->stop_after_group = -1;
  for (uint32_t gi = 0; gi < s->c_group_cnt[c]; gi++) memset(&x->out->groups[s->c_group_off[c] + gi], 0, sizeof(kr_group_result));
  /* a context is reused across runs: this cluster's pods start without an action */
  for (uint32_t i = x->cl_start[c]; i < x->cl_start[c + 1]; i++) x->act[x->cl_pods[i]] = KR_ACT_KEEP;
  char *h = x->out->hash + 32 * (size_t)c;
  /* :623 — computed every reconcile */
  if (x->f->skip_hash) memset(h, 0, 32);
  else kr_oracle_hash32(s->json + s->c_json_off[c], s->c_json_len[c], h);
  uint32_t cf = s->c_flags[c];
  if (cf & KR_CF_SKIP) { cr->path = KR_PATH_SKIPPED; return; }
  if (s->c_ext_err_kind[c] != KR_EXT_ERR_NONE) { /* an earlier sub-reconciler failed: reconcilePods not reached (:308-314) */
    cr->path = KR_PATH_SKIPPED;
    cr->err_kind = s->c_ext_err_kind[c] == KR_EXT_ERR_STATUS_ONLY_NIL ? KR_ERR_NONE : KR_ERR_EXTERNAL;
  } else {
    reconcile_pods(x, t, c, h, cr, creates);
  }
  calculate_status(x, t, c, cr);
}

static void *worker_main(void *p) {
  worker_arg *a = (worker_arg *)p;
  oscratch t; memset(&t, 0, sizeof t);
  for (int r = 0; r < a->reps; r++) {
    a->creates.n = 0;
    for (uint32_t c = a->c0; c < a->c1; c++) reconcile_cluster(a->x, &t, c, &a->creates);
  }
  scratch_free(&t);
  return NULL;
}

static int build_context(octx *x) {
  const kr_snapshot_bufs *s = x->s; const kr_sizes *n = x->n;
  uint32_t Nc = n->n_clusters, Np = n->n_pods;
  if (kmap_init(&x->cluster_map, Nc) || kmap_init(&x->podname_map, Np) || kmap_init(&x->ns_map, Np + Nc)) return KR_E_CAPACITY;
  for (uint32_t c = 0; c < Nc; c++) kmap_put_first(&x->cluster_map, key2(s->c_ns_id[c], s->c_name_id[c]), c);
  x->pod_cluster = (uint32_t *)malloc(((size_t)Np + 1) * 4);
  x->cl_start = (uint32_t *)calloc((size_t)Nc + 3, 4);
  x->cl_pods = (uint32_t *)malloc(((size_t)Np + 1) * 4);
  x->ns_pods = (uint32_t *)malloc(((size_t)Np + 1) * 4);
  x->pod_head_aux = (int32_t *)malloc(((size_t)Np + 1) * 4);
  x->act = (uint8_t *)calloc((size_t)Np + 1, 1);
  /* namespaces -> dense buckets */
  uint32_t Nns = 0;
  for (uint32_t p = 0; p < Np; p++) { uint32_t b; if (!kmap_get(&x->ns_map, s->p_ns_id[p], &b)) kmap_put_first(&x->ns_map, s->p_ns_id[p], Nns++); }
  for (uint32_t c = 0; c < Nc; c++) { uint32_t b; if (!kmap_get(&x->ns_map, s->c_ns_id[c], &b)) kmap_put_first(&x->ns_map, s->c_ns_id[c], Nns++); }
  x->ns_start = (uint32_t *)calloc((size_t)Nns + 2, 4);
  for (uint32_t p = 0; p < Np; p++) {
    uint32_t c = Nc;
    if (s->p_cluster_name_id[p] != 0) { uint32_t v; if (kmap_get(&x->cluster_map, key2(s->p_ns_id[p], s->p_cluster_name_id[p]), &v)) c = v; }
    x->pod_cluster[p] = c; x->cl_start[c + 1]++;
    uint32_t b = 0; kmap_get(&x->ns_map, s->p_ns_id[p], &b); x->ns_start[b + 1]++;
    kmap_put_first(&x->podname_map, key2(s->p_ns_id[p], s->p_name_id[p]), p);
    x->pod_head_aux[p] = -1;
  }
  for (uint32_t c = 0; c <= Nc; c++) x->cl_start[c + 1] += x->cl_start[c];
  for (uint32_t b = 0; b < Nns; b++) x->ns_start[b + 1] += x->ns_start[b];
  uint32_t *cw = (uint32_t *)malloc(((size_t)Nc + 2) * 4), *nw = (uint32_t *)malloc(((size_t)Nns + 1) * 4);
  memcpy(cw, x->cl_start, ((size_t)Nc + 2) * 4); memcpy(nw, x->ns_start, ((size_t)Nns + 1) * 4);
  for (uint32_t p = 0; p < Np; p++) {
    x->cl_pods[cw[x->pod_cluster[p]]++] = p;
    uint32_t b = 0; kmap_get(&x->ns_map, s->p_ns_id[p], &b); x->ns_pods[nw[b]++] = p;
  }
  free(cw); free(nw);
  for (uint32_t h = 0; h < n->n_heads; h++) {
    uint32_t p = s->h_pod_idx[h];
    if (p < Np && x->pod_head_aux[p] < 0) x->pod_head_aux[p] = (int32_t)h;
  }
  /* resolve WorkersToDelete names: Delete(ns of the cluster, name) (:818-822) */
  x->wtd = (int32_t *)malloc(((size_t)n->n_wtd + 1) * 4);
  for (uint32_t g = 0; g < n->n_groups; g++) {
    uint32_t c = s->g_cluster_idx[g];
    for (uint32_t w = 0; w < s->g_wtd_cnt[g]; w++) {
      uint32_t e = s->g_wtd_off[g] + w, v;
      x->wtd[e] = kmap_get(&x->podname_map, key2(s->c_ns_id[c], s->w_name_id[e]), &v) ? (int32_t)v : -1;
    }
  }
  return 0;
}

static void free_context(octx *x) {
  kmap_free(&x->cluster_map); kmap_free(&x->podname_map); kmap_free(&x->ns_map);
  free(x->pod_cluster); free(x->cl_start); free(x->cl_pods); free(x->ns_start); free(x->ns_pods); free(x->pod_head_aux); free(x->wtd); free(x->act);
}

/* The shared index of one snapshot: what controller-runtime's informer cache holds between reconciles (its namespace index is
 * maintained incrementally from watch events, never rebuilt per List).  Built once per snapshot, reused by every run. */
struct kr_oracle_ctx { octx x; kr_sizes n; };

int kr_oracle_ctx_create(const kr_snapshot_bufs *s, const kr_sizes *n, kr_oracle_ctx **out) {
  if (!s || !n || !out) return KR_E_INVALID;
  kr_oracle_ctx *cx = (kr_oracle_ctx *)calloc(1, sizeof *cx);
  if (!cx) return KR_E_CAPACITY;
  cx->n = *n;
  cx->x.s = s; cx->x.n = &cx->n;
  int rc = build_context(&cx->x);
  if (rc) { free_context(&cx->x); free(cx); return rc; }
  *out = cx;
  return 0;
}

void kr_oracle_ctx_destroy(kr_oracle_ctx *cx) {
  if (!cx) return;
  free_context(&cx->x);
  free(cx);
}

static int ctx_run(kr_oracle_ctx *cx, const kr_flags *f, kr_oracle_out *out, int list_mode, int threads, uint32_t c0, uint32_t c1, int reps, int full) {
  octx *x = &cx->x;
  const kr_snapshot_bufs *s = x->s; const kr_sizes *n = x->n;
  x->f = f; x->out = out; x->list_mode = list_mode;
  if (c1 > n->n_clusters) c1 = n->n_clusters;
  if (reps < 1) reps = 1;
  int rc = 0;
  if (n->n_wtd) memcpy(out->wtd_pod_idx, x->wtd, (size_t)n->n_wtd * 4);
  if (threads < 1) threads = 1;
  uint32_t span = c1 > c0 ? c1 - c0 : 0;
  if ((uint32_t)threads > span) threads = span ? (int)span : 1;
  worker_arg *args = (worker_arg *)calloc((size_t)threads, sizeof(worker_arg));
  pthread_t *tids = (pthread_t *)calloc((size_t)threads, sizeof(pthread_t));
  for (int t = 0; t < threads; t++) {
    args[t].x = x; args[t].reps = reps;
    args[t].c0 = c0 + (uint32_t)(((uint64_t)span * t) / threads);
    args[t].c1 = c0 + (uint32_t)(((uint64_t)span * (t + 1)) / threads);
    if (threads == 1) worker_main(&args[t]);
    else pthread_create(&tids[t], NULL, worker_main, &args[t]);
  }
  if (threads > 1) for (int t = 0; t < threads; t++) pthread_join(tids[t], NULL);

  if (full) {
    /* RayJob roll-up: rayjob_controller.go:203-216 (getOrCreateRayClusterInstance + state gate), :343, :885 */
    for (uint32_t j = 0; j < n->n_jobs; j++) {
      kr_job_result *jr = &out->jobs[j];
      memset(jr, 0, sizeof *jr);
      uint32_t c;
      if (s->j_cluster_name_id[j] == 0 || !kmap_get(&x->cluster_map, key2(s->j_ns_id[j], s->j_cluster_name_id[j]), &c)) { jr->cluster_idx = -1; continue; }
      jr->cluster_idx = (int32_t)c;
      jr->cluster_state = s->c_old_state[c];
      jr->not_ready = s->c_old_state[c] != KR_STATE_READY;
      jr->status_changed = s->j_summary_id[j] != s->c_summary_id[c];
    }
    /* create arena: groups in global order (workers ran over ascending cluster ranges, so streams are ordered) */
    uint32_t total = 0;
    for (int t = 0; t < threads && rc == 0; t++) {
      ivec *cv = &args[t].creates;
      for (uint32_t i = 0; i < cv->n;) {
        uint32_t cnt = (uint32_t)cv->v[i + 1];
        if ((uint64_t)total + cnt > out->create_cap) { rc = KR_E_CAPACITY; break; }
        memcpy(out->create_idx + total, cv->v + i + 2, cnt * sizeof(int32_t));
        total += cnt; i += 2 + cnt;
      }
    }
    out->n_create_total = total;
    /* groups without creates: create_off = running total position (exclusive scan of n_create) */
    uint32_t run = 0;
    for (uint32_t g = 0; g < n->n_groups; g++) { out->groups[g].create_off = run; run += out->groups[g].n_create; }
    /* pods bucketed by cluster, list order; orphans last */
    uint32_t Nc = n->n_clusters, n_actions = 0, n_tomb = 0;
    for (uint32_t i = 0; i < n->n_pods; i++) {
      uint32_t p = x->cl_pods[i];
      out->sorted_pod_idx[i] = p;
      uint8_t a = x->pod_cluster[p] == Nc ? ((s->p_packed[p] & KR_PP_TOMBSTONE) ? KR_ACT_TOMBSTONE : KR_ACT_ORPHAN) : x->act[p];
      out->sorted_action[i] = a;
      if (a == KR_ACT_TOMBSTONE) n_tomb++;
      if (a != KR_ACT_KEEP && a != KR_ACT_ORPHAN && a != KR_ACT_TOMBSTONE) n_actions++;
    }
    for (uint32_t c = 0; c < Nc; c++) out->clusters[c].pod_start = x->cl_start[c];
    /* compact action list, cluster-major, list order inside a cluster */
    uint32_t na = 0;
    for (uint32_t c = 0; c < Nc; c++) {
      out->act_start[c] = na;
      for (uint32_t i = x->cl_start[c]; i < x->cl_start[c + 1]; i++) {
        uint8_t a = x->act[x->cl_pods[i]];
        if (a != KR_ACT_KEEP) { out->act_pod_idx[na] = x->cl_pods[i]; out->act_code[na] = a; na++; }
      }
    }
    out->act_start[Nc] = na;
    for (uint32_t c = 0; c < Nc; c++) out->act_cnt[c] = out->act_start[c + 1] - out->act_start[c];
    out->n_orphans = x->cl_start[Nc + 1] - x->cl_start[Nc] - n_tomb;  /* free rows sit in the orphans' segment but are not orphans */
    out->n_actions = n_actions;
  }
  for (int t = 0; t < threads; t++) free(args[t].creates.v);
  free(args); free(tids);
  return rc;
}

int kr_oracle_ctx_run(kr_oracle_ctx *cx, const kr_flags *f, kr_oracle_out *out, int list_mode, int threads) {
  if (!cx || !f || !out) return KR_E_INVALID;
  return ctx_run(cx, f, out, list_mode, threads, 0, cx->n.n_clusters, 1, 1);
}

int kr_oracle_ctx_run_range(kr_oracle_ctx *cx, const kr_flags *f, kr_oracle_out *out, int list_mode, int threads,
                            uint32_t c0, uint32_t c1, int reps) {
  if (!cx || !f || !out) return KR_E_INVALID;
  return ctx_run(cx, f, out, list_mode, threads, c0, c1, reps, 0);
}

int kr_oracle_run(const kr_snapshot_bufs *s, const kr_sizes *n, const kr_flags *f, kr_oracle_out *out, int list_mode, int threads) {
  kr_oracle_ctx *cx = NULL;
  int rc = kr_oracle_ctx_create(s, n, &cx);
  if (rc) return rc;
  rc = kr_oracle_ctx_run(cx, f, out, list_mode, threads);
  kr_oracle_ctx_destroy(cx);
  return rc;
}

int kr_oracle_run_range(const kr_snapshot_bufs *s, const kr_sizes *n, const kr_flags *f, kr_oracle_out *out,
                        int list_mode, int threads, uint32_t c0, uint32_t c1) {
  kr_oracle_ctx *cx = NULL;
  int rc = kr_oracle_ctx_create(s, n, &cx);
  if (rc) return rc;
  rc = kr_oracle_ctx_run_range(cx, f, out, list_mode, threads, c0, c1, 1);
  kr_oracle_ctx_destroy(cx);
  return rc;
}
