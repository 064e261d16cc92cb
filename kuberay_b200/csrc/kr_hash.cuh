// kr_hash.cuh — SHA-1 + base32hex of the muted-spec JSON (GenerateJsonHash, utils/util.go:628-640).
// Part of the sm_90a kernel set of the batched reconcile engine; see kr_kernels.cuh for the pipeline overview.
#pragma once

#include "kr_common.cuh"

namespace kr {

// ------------------------------------------------------------------------------------------------ k_hash
// base32hex(sha1(json)) per RayCluster (utils/util.go:628-640).  One lane per message (SHA-1 is a serial chain per
// message); the warp stages 128 bytes of each of its 32 messages per step with coalesced 16-byte loads into an
// XOR-swizzled shared tile, so the per-lane reads are conflict-free LDS.128.

__device__ __forceinline__ uint32_t rol(uint32_t x, int k) { return __funnelshift_l(x, x, k); }
__device__ __forceinline__ uint32_t bswap(uint32_t x) { return __byte_perm(x, 0, 0x0123); }

// ------------------------------------------------------------------------------------------------ k_hash2
// Second-generation hash kernel.  Same one-lane-per-message mapping, but
//  (1) the 128-byte chunks are fetched with cp.async (LDGSTS) straight into a double-buffered, XOR-swizzled shared tile:
//      no register staging, and the fetch of chunk i+1 is in flight during the 160 rounds of chunk i by construction;
//  (2) each round is written so that the only operation on the serial a->a chain is rol5(a)+s (one LEA.HI); s = f+e+K+w is
//      formed off the chain;
//  (3) VARIANT 1 forms s with IMADs (multiply by an opaque 1 from the constant bank) so those adds issue on the FMA pipe
//      while LOP3/SHF/LEA keep the ALU pipe.  tools/hash_bench.cu times the variants: with one
//      warp per scheduler (10k messages) VARIANT 0 is the one to use (8 ALU-pipe instructions per round at 2 cycles each is
//      the floor), with many warps per scheduler (100k messages) VARIANT 1.
__device__ __forceinline__ void cp_async16(void *smem_dst, const void *gsrc, uint32_t src_bytes) {
  uint32_t d = (uint32_t)__cvta_generic_to_shared(smem_dst);
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(d), "l"(gsrc), "r"(src_bytes) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N> __device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

__device__ __forceinline__ uint32_t mad1(uint32_t a, uint32_t one, uint32_t c) {
  uint32_t d;
  asm("mad.lo.u32 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(one), "r"(c));
  return d;
}

// rol(x, n) on the FMA pipe: x * 2^n as a 64-bit product puts x << n in the low word and x >> (32 - n) in the high word; the
// two halves have no bit in common, so lo * 1 + hi is the rotation.  `pow2` and `one` are opaque (derived from a kernel
// parameter), otherwise ptxas strength-reduces both back to ALU-pipe shifts.
__device__ __forceinline__ uint32_t rol_fma(uint32_t x, uint32_t pow2, uint32_t one) {
  uint32_t r;
  asm("{\n\t.reg .u64 t;\n\t.reg .u32 lo, hi;\n\tmul.wide.u32 t, %1, %2;\n\tmov.b64 {lo, hi}, t;\n\tmad.lo.u32 %0, lo, %3, hi;\n\t}" : "=r"(r) : "r"(x), "r"(pow2), "r"(one));
  return r;
}

// VARIANT: 0 = every round operation on the ALU pipe; 1 = s formed by two IMADs; 2..5 = experiments that move off-chain work
// to the FMA pipe (5: w+K; 2: w+K and rol30(b); 3: w+K and the schedule's rol1; 4: all three) hoping a lone warp would
// alternate pipes.  It did not pay: at 10k messages
// each of 2..5 was slower than 0, at 100k messages only VARIANT 1 beat 0.  The engine uses 0 (latency regime) and 1 (throughput
// regime); 2..5 stay for tools/hash_bench.cu, which times them all.
template <int VARIANT>
__device__ __forceinline__ void sha1_rounds2(uint32_t (&w)[16], uint32_t (&h)[5], uint32_t one) {
  uint32_t a = h[0], b = h[1], c = h[2], d = h[3], e = h[4];
  const uint32_t two = one << 1, two30 = one << 30;
  constexpr bool kFmaRol30 = VARIANT == 2 || VARIANT == 4, kFmaRol1 = VARIANT == 3 || VARIANT == 4;
#pragma unroll
  for (int i = 0; i < 80; i++) {
    uint32_t wi;
    if (i < 16) wi = w[i];
    else {
      const uint32_t x = w[(i - 3) & 15] ^ w[(i - 8) & 15] ^ w[(i - 14) & 15] ^ w[i & 15];
      wi = kFmaRol1 ? rol_fma(x, two, one) : rol(x, 1);
      w[i & 15] = wi;
    }
    const uint32_t k = i < 20 ? 0x5A827999u : (i < 40 ? 0x6ED9EBA1u : (i < 60 ? 0x8F1BBCDCu : 0xCA62C1D6u));
    uint32_t f;
    if (i < 20) f = (b & c) | (~b & d);
    else if (i < 40) f = b ^ c ^ d;
    else if (i < 60) f = (b & c) | (b & d) | (c & d);
    else f = b ^ c ^ d;
    uint32_t s;
    if (VARIANT == 0) s = f + e + (wi + k);            // lone warp per scheduler (latency regime): fewest instructions wins
    else if (VARIANT == 1) s = mad1(f, one, mad1(e, one, wi + k));  // many warps per scheduler (throughput regime): adds on the FMA pipe
    else s = f + e + mad1(wi, one, k);                  // w + K is far off the chain: FMA pipe
    asm volatile("" : "+r"(s));  // keep s a value of its own: the a->a chain below is then a single rol5(a)+s
    uint32_t t = rol(a, 5) + s;
    e = d; d = c; c = kFmaRol30 ? rol_fma(b, two30, one) : rol(b, 30); b = a; a = t;
  }
  h[0] += a; h[1] += b; h[2] += c; h[3] += d; h[4] += e;
}

// SHA-1 state -> the 32 base32hex characters of the digest (no padding: 160 bits are exactly 32 characters).
__device__ __forceinline__ void digest_to_base32hex(const uint32_t (&h)[5], char *__restrict__ out32) {
  uint32_t o32[8];
#pragma unroll
  for (int j = 0; j < 4; j++) {
    uint64_t v;
    switch (j) {
      case 0: v = ((uint64_t)h[0] << 8) | (h[1] >> 24); break;
      case 1: v = ((uint64_t)(h[1] & 0xFFFFFFu) << 16) | (h[2] >> 16); break;
      case 2: v = ((uint64_t)(h[2] & 0xFFFFu) << 24) | (h[3] >> 8); break;
      default: v = ((uint64_t)(h[3] & 0xFFu) << 32) | h[4]; break;
    }
    uint32_t lo = 0, hi = 0;
#pragma unroll
    for (int kk = 0; kk < 8; kk++) {
      const uint32_t cc = (uint32_t)(v >> (35 - 5 * kk)) & 31u;
      const uint32_t ch = cc < 10 ? ('0' + cc) : ('A' + cc - 10);
      if (kk < 4) lo |= ch << (8 * kk); else hi |= ch << (8 * (kk - 4));
    }
    o32[2 * j] = lo; o32[2 * j + 1] = hi;
  }
  // The last word is the digest's "ready" mark: a decide warp of the concurrently running main chain may be polling it
  // (k_decide2: Recreate gate), so both hash kernels (k_hash2, k_hash3) store it after a fence, once the other 28 bytes are
  // visible.
  uint4 *dst = reinterpret_cast<uint4 *>(out32);
  dst[0] = make_uint4(o32[0], o32[1], o32[2], o32[3]);
  reinterpret_cast<uint2 *>(out32)[2] = make_uint2(o32[4], o32[5]);
  reinterpret_cast<uint32_t *>(out32)[6] = o32[6];
  __threadfence();
  reinterpret_cast<volatile uint32_t *>(out32)[7] = o32[7];
}

template <int WARPS, int VARIANT>
__global__ void __launch_bounds__(WARPS * 32) k_hash2(const uint8_t *__restrict__ bytes, const uint64_t *__restrict__ off,
                                                      const uint32_t *__restrict__ len32, const uint32_t *__restrict__ order,
                                                      uint32_t n, char *__restrict__ out, uint32_t one = 1) {
  KR_TL(7);
  __shared__ uint4 s_tile[2][WARPS][32][8];  // [buffer][warp][message lane][16-byte piece ^ (lane & 7)]
  const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  // grid-stride over groups of WARPS*32 messages: the engine caps the grid for large n so that the hash leaves room on every
  // SM for the main chain's blocks (each warp owns its shared tile, so the trips need no block-wide barrier)
  for (uint32_t grp_i = blockIdx.x; (uint64_t)grp_i * (WARPS * 32) < n; grp_i += gridDim.x) {
  const uint32_t slot_i = (grp_i * WARPS + warp) * 32 + lane;
  const bool have = slot_i < n;
  const uint32_t m = have ? (order ? __ldg(&order[slot_i]) : slot_i) : 0u;  // `order`: message ids by descending block count (length-homogeneous warps)
  uint64_t moff = 0;
  uint32_t mlen = 0;
  if (have) { moff = off[m]; mlen = len32[m]; }
  const uint32_t nblocks = have ? (mlen + 8) / 64 + 1 : 0;
  uint32_t max_blocks = nblocks;
#pragma unroll
  for (int d = 16; d; d >>= 1) max_blocks = max(max_blocks, __shfl_xor_sync(0xFFFFFFFFu, max_blocks, d));
  uint32_t h[5] = {0x67452301u, 0xEFCDAB89u, 0x98BADCFEu, 0x10325476u, 0xC3D2E1F0u};
  const uint32_t sub = lane & 7, grp = lane >> 3;
  // this lane fetches piece `sub` of messages 4r+grp, r = 0..7: keep their base pointers and padded lengths
  const uint8_t *src[8];
  uint32_t lim[8];
#pragma unroll
  for (int r = 0; r < 8; r++) {
    uint32_t sl = 4 * r + grp;
    uint64_t o = __shfl_sync(0xFFFFFFFFu, moff, sl);
    uint32_t l = __shfl_sync(0xFFFFFFFFu, mlen, sl);
    src[r] = bytes + o + sub * 16;
    lim[r] = (l + 15) & ~15u;  // the arena pads every message to 16 bytes
  }
  auto fetch = [&](uint32_t chunk, int buf) {
#pragma unroll
    for (int r = 0; r < 8; r++) {
      uint32_t sl = 4 * r + grp;
      uint32_t pos = chunk * 128 + sub * 16;
      bool in = pos < lim[r];
      cp_async16(&s_tile[buf][warp][sl][sub ^ (sl & 7)], in ? (const void *)(src[r] + (size_t)chunk * 128) : (const void *)bytes, in ? 16u : 0u);
    }
    cp_async_commit();
  };
  const uint32_t nchunks = (max_blocks + 1) / 2;
  if (nchunks) fetch(0, 0);
  for (uint32_t chunk = 0; chunk < nchunks; chunk++) {
    const int buf = chunk & 1;
    if (chunk + 1 < nchunks) { fetch(chunk + 1, buf ^ 1); cp_async_wait<1>(); }
    else cp_async_wait<0>();
    __syncwarp();
#pragma unroll
    for (int half = 0; half < 2; half++) {
      uint32_t blk = chunk * 2 + half;
      if (blk >= nblocks) continue;
      uint32_t w[16];
#pragma unroll
      for (int q = 0; q < 4; q++) {
        uint4 v = s_tile[buf][warp][lane][(half * 4 + q) ^ (lane & 7)];
        w[4 * q] = bswap(v.x); w[4 * q + 1] = bswap(v.y); w[4 * q + 2] = bswap(v.z); w[4 * q + 3] = bswap(v.w);
      }
      const uint32_t bstart = blk * 64;
      if (bstart + 64 > mlen) {  // tail block(s): 0x80, zero fill, 64-bit big-endian bit length (FIPS 180-4 §5.1.1)
#pragma unroll
        for (int q = 0; q < 16; q++) {
          uint32_t wpos = bstart + 4 * q;
          uint32_t v = w[q];
          if (wpos >= mlen) v = (wpos == mlen) ? 0x80000000u : 0u;
          else if (wpos + 4 > mlen) {
            uint32_t keep = mlen - wpos;  // 1..3 message bytes in this word
            v = (v & (0xFFFFFFFFu << (8 * (4 - keep)))) | (0x80u << (8 * (3 - keep)));
          }
          w[q] = v;
        }
        if (blk == nblocks - 1) { w[14] = mlen >> 29; w[15] = mlen << 3; }
      }
      sha1_rounds2<VARIANT>(w, h, one);
    }
    __syncwarp();  // every lane is done reading this buffer before the fetch two iterations ahead overwrites it
  }
  if (have) digest_to_base32hex(h, out + 32 * (size_t)m);
  __syncwarp();
  }  // next group of messages
}

// ------------------------------------------------------------------------------------------------ k_hash3
// Third-generation hash kernel: the SHA-1 round chain and everything that is NOT on it run on different warp schedulers.
//
//   producer warp  stages 128 bytes of each of its 32 messages per step with cp.async (LDGSTS.128, double-buffered, XOR-swizzled
//                  tile), byte-swaps, applies the FIPS 180-4 padding, expands the message schedule W[16..79] and adds the round
//                  constants: 80 ready-to-use words wk[t] = W[t] + K[t] per 64-byte block, written to a 3-stage ring;
//                  (a 1-D bulk copy per message — cp.async.bulk / UBLKCP — was built and dropped: UBLKCP takes warp-uniform
//                  operands, so 32 per-lane sources compile to a 32-trip serialised loop of ~13 instructions, 208 instructions
//                  per block against 4 for the LDGSTS form)
//   consumer warp  lane L runs only the serial a->a chain of message L: per round f (LOP3), f+e+wk (IADD3), rol5(a)+s (LEA.HI),
//                  rol30(b) (SHF) — 4 ALU-pipe instructions instead of the 8.6 of the single-warp kernel — reading wk with LDS.128.
//
// The two warps of a pair sit on different schedulers of the SM (warp id within the CTA selects the sub-partition), hand
// blocks over through named barriers (full / empty per ring stage), and a CTA is one pair, so a 10 k-message snapshot (313 groups
// of 32 messages) puts one hash warp on every scheduler of the chip instead of one 8.6-instruction-per-round warp on half of them.
// `order` lists the message ids by descending block count (built by the host at commit, which knows c_json_len): warps are
// length-homogeneous — the unsorted kernel ran every warp to its longest message, 42 % idle lane-rounds on the 1.5/2.5/4/6 KB
// mix — and groups are dealt to the CTAs longest first, snaking (0..G-1, G-1..0, ...), so every CTA gets about the same work.
// The wk rows are padded to 336 B (and the raw tile swizzled) so that the per-lane 16-byte accesses of a quarter warp fall in
// distinct banks.
static constexpr int kH3WkStride = 84;    // u32 per message row of a wk stage: 80 words + 4 pad

static constexpr int kH3Stages = 3;       // wk ring depth
struct H3Smem {
  uint4 raw[2][32][8];                   // [stage][message lane][16-byte piece ^ (lane & 7)] — the XOR-swizzled tile of k_hash2
  uint32_t wk[kH3Stages][32][kH3WkStride];
};
// full / empty hand-offs of a ring stage between the two warps of a pair: hardware named barriers (bar.arrive by the signalling
// warp, bar.sync by the waiting one, 64 participants).  mbarrier arrive -> try_wait was tried first and costs several
// times the barrier unit's latency per direction (tools/hash_bench MODE 3 times the ping-pong alone).
__device__ __forceinline__ void nbar_arrive(uint32_t id) { asm volatile("bar.arrive %0, 64;" ::"r"(id) : "memory"); }
__device__ __forceinline__ void nbar_sync(uint32_t id) { asm volatile("bar.sync %0, 64;" ::"r"(id) : "memory"); }

// the chain: 80 rounds over one block's wk words (consumer warp).  ptxas pairs the rounds (LEA.HI t, SHF, LEA.HI t', SHF, LOP3 f,
// LOP3 f', IADD3 s, IADD3 s'): 4.25 ALU-pipe instructions per round, every one two issue slots behind its producer.  For a lone
// warp (tools/hash_bench, MODE 4) the f -> s -> t dependency path (3 dependent ALU
// operations per 2 rounds at ~8 cycles each), not the issue rate, is the floor; a source-level software pipeline (f', s' of round
// i+1 before t of round i) is rescheduled by ptxas into the same pairs.
__device__ __forceinline__ void sha1_chain80(const uint32_t *__restrict__ wk /* this lane's row of the stage */, uint32_t (&h)[5]) {
  uint32_t a = h[0], b = h[1], c = h[2], d = h[3], e = h[4];
#pragma unroll
  for (int q = 0; q < 20; q++) {
    const uint4 v = *reinterpret_cast<const uint4 *>(wk + 4 * q);
    const uint32_t ww[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
    for (int j = 0; j < 4; j++) {
      const int i = 4 * q + j;
      uint32_t f;
      if (i < 20) f = (b & c) | (~b & d);
      else if (i < 40) f = b ^ c ^ d;
      else if (i < 60) f = (b & c) | (b & d) | (c & d);
      else f = b ^ c ^ d;
      uint32_t s = f + e + ww[j];
      asm volatile("" : "+r"(s));  // keep s a value of its own: the a->a chain is then a single rol5(a)+s
      const uint32_t t = rol(a, 5) + s;
      e = d; d = c; c = rol(b, 30); b = a; a = t;
    }
  }
  h[0] += a; h[1] += b; h[2] += c; h[3] += d; h[4] += e;
}

// one 64-byte block of this lane's message: raw bytes -> wk[0..79] (producer warp)
__device__ __forceinline__ void sha1_expand_block(const uint4 *__restrict__ tile_row /* this lane's 8 swizzled pieces */, int half, uint32_t lane,
                                                  uint32_t *__restrict__ wk_row, uint32_t blk, uint32_t nblocks, uint32_t mlen) {
  uint32_t w[16];
#pragma unroll
  for (int q = 0; q < 4; q++) {
    const uint4 v = tile_row[(half * 4 + q) ^ (lane & 7)];
    w[4 * q] = bswap(v.x); w[4 * q + 1] = bswap(v.y); w[4 * q + 2] = bswap(v.z); w[4 * q + 3] = bswap(v.w);
  }
  const uint32_t bstart = blk * 64;
  if (bstart + 64 > mlen) {  // tail block(s): 0x80, zero fill, 64-bit big-endian bit length (FIPS 180-4 §5.1.1)
#pragma unroll
    for (int q = 0; q < 16; q++) {
      const uint32_t wpos = bstart + 4 * q;
      uint32_t v = w[q];
      if (wpos >= mlen) v = (wpos == mlen) ? 0x80000000u : 0u;
      else if (wpos + 4 > mlen) {
        const uint32_t keep = mlen - wpos;  // 1..3 message bytes in this word
        v = (v & (0xFFFFFFFFu << (8 * (4 - keep)))) | (0x80u << (8 * (3 - keep)));
      }
      w[q] = v;
    }
    if (blk == nblocks - 1) { w[14] = mlen >> 29; w[15] = mlen << 3; }
  }
  // W[i] = rol1(W[i-3] ^ X[i]) with X[i] = W[i-8] ^ W[i-14] ^ W[i-16]: X only needs words at least 8 back, so it is formed three
  // words ahead and kept opaque — the recurrence through W[i-3] is then LOP3 + SHF (two dependent ALU operations per three words)
  // instead of the LOP3 + LOP3 + SHF ptxas builds when it is free to re-associate the four-way XOR.
  uint32_t x[3];
#pragma unroll
  for (int i = 16; i < 19; i++) { x[i % 3] = w[(i - 8) & 15] ^ w[(i - 14) & 15] ^ w[i & 15]; asm volatile("" : "+r"(x[i % 3])); }
#pragma unroll
  for (int q = 0; q < 20; q++) {
    uint32_t o[4];
#pragma unroll
    for (int j = 0; j < 4; j++) {
      const int i = 4 * q + j;
      uint32_t wi;
      if (i < 16) wi = w[i];
      else {
        wi = rol(w[(i - 3) & 15] ^ x[i % 3], 1);
        w[i & 15] = wi;
        if (i + 3 < 80) { x[i % 3] = w[(i + 3 - 8) & 15] ^ w[(i + 3 - 14) & 15] ^ w[(i + 3) & 15]; asm volatile("" : "+r"(x[i % 3])); }
      }
      const uint32_t k = i < 20 ? 0x5A827999u : (i < 40 ? 0x6ED9EBA1u : (i < 60 ? 0x8F1BBCDCu : 0xCA62C1D6u));
      o[j] = wi + k;
    }
    *reinterpret_cast<uint4 *>(wk_row + 4 * q) = make_uint4(o[0], o[1], o[2], o[3]);
  }
}

// grid: CTAs of PAIRS x 64 threads (even warp = consumer, odd warp = producer); G = total pairs; group g of 32 messages (in
// `order`) goes to pair (g % G) on even rounds and G-1-(g % G) on odd ones.
// PAIRS consumer/producer pairs per CTA (warps 2p and 2p+1).  MODE (tools/hash_bench.cu only): 1 = the consumer skips the rounds,
// 2 = the producer skips the expansion, 3 = both skip (hand-off cost alone), 4 = no hand-offs (compute alone); the engine uses MODE 0.
template <int PAIRS, int MODE>
__global__ void __launch_bounds__(PAIRS * 64) k_hash3(const uint8_t *__restrict__ bytes, const uint64_t *__restrict__ off, const uint32_t *__restrict__ len32,
                                                      const uint32_t *__restrict__ order, uint32_t n, char *__restrict__ out) {
  KR_TL(7);
  extern __shared__ __align__(16) uint8_t h3_dyn[];  // PAIRS x H3Smem (PAIRS = 2 is above the 48 KB static limit)
  H3Smem *sm_all = reinterpret_cast<H3Smem *>(h3_dyn);
  const uint32_t pair = threadIdx.x >> 6, warp = (threadIdx.x >> 5) & 1, lane = threadIdx.x & 31;
  H3Smem &sm = sm_all[pair];
  // named barriers of this pair: 1 + pair * 2 * kH3Stages + {stage (full), kH3Stages + stage (empty)}
  const uint32_t bar0 = 1 + pair * 2 * kH3Stages;
  static_assert(1 + PAIRS * 2 * kH3Stages <= 16, "16 named barriers per CTA");
  const uint32_t ngroups = (n + 31) / 32, G = gridDim.x * PAIRS, me = blockIdx.x * PAIRS + pair;
  uint32_t chunk_seq = 0, blk_seq = 0;  // running use counts of the raw stages / wk stages (same in both warps)
  for (uint32_t round = 0;; round++) {
    const uint32_t g = round * G + ((round & 1) ? G - 1 - me : me);
    if (round * G >= ngroups) break;
    if (g >= ngroups) continue;
    const uint32_t slot = g * 32 + lane;
    const bool have = slot < n;
    const uint32_t m = have ? (order ? __ldg(&order[slot]) : slot) : 0u;
    uint64_t moff = 0;
    uint32_t mlen = 0;
    if (have) { moff = __ldg(&off[m]); mlen = __ldg(&len32[m]); }
    const uint32_t nblocks = have ? (mlen + 8) / 64 + 1 : 0;
    const uint32_t max_blocks = __reduce_max_sync(0xFFFFFFFFu, nblocks);
    const uint32_t nchunks = (max_blocks + 1) / 2;
    if (warp == 1) {
      // ---------------- producer
      // this lane fetches piece `sub` of messages 4r+grp, r = 0..7 (8 lanes cover one message's 128 bytes: coalesced)
      const uint32_t sub = lane & 7, grp = lane >> 3;
      const uint8_t *src[8];
      uint32_t lim[8];
#pragma unroll
      for (int r = 0; r < 8; r++) {
        const uint32_t sl = 4 * r + grp;
        const uint64_t o = __shfl_sync(0xFFFFFFFFu, moff, sl);
        const uint32_t l = __shfl_sync(0xFFFFFFFFu, mlen, sl);
        src[r] = bytes + o + sub * 16;
        lim[r] = (l + 15) & ~15u;  // the arena pads every message to 16 bytes
      }
      auto fetch = [&](uint32_t chunk, uint32_t buf) {
#pragma unroll
        for (int r = 0; r < 8; r++) {
          const uint32_t sl = 4 * r + grp;
          const bool in = chunk * 128 + sub * 16 < lim[r];
          cp_async16(&sm.raw[buf][sl][sub ^ (sl & 7)], in ? (const void *)(src[r] + (size_t)chunk * 128) : (const void *)bytes, in ? 16u : 0u);
        }
        cp_async_commit();
      };
      if (nchunks) fetch(0, chunk_seq & 1);
      for (uint32_t chunk = 0; chunk < nchunks; chunk++) {
        const uint32_t buf = (chunk_seq + chunk) & 1;
        if (chunk + 1 < nchunks) { fetch(chunk + 1, buf ^ 1); cp_async_wait<1>(); }
        else cp_async_wait<0>();
        __syncwarp();
#pragma unroll
        for (int half = 0; half < 2; half++) {
          const uint32_t blk = chunk * 2 + half;
          if (blk >= max_blocks) break;
          const uint32_t bs = blk_seq + blk, stage = bs % kH3Stages;
          if (MODE != 4 && bs >= kH3Stages) nbar_sync(bar0 + kH3Stages + stage);  // the consumer has left this stage
          if (MODE != 2 && MODE != 3 && blk < nblocks) sha1_expand_block(&sm.raw[buf][lane][0], half, lane, &sm.wk[stage][lane][0], blk, nblocks, mlen);
          if (MODE != 4) nbar_arrive(bar0 + stage);
        }
        __syncwarp();  // every lane is done reading this raw stage before the fetch two iterations ahead overwrites it
      }
    } else {
      // ---------------- consumer
      uint32_t h[5] = {0x67452301u, 0xEFCDAB89u, 0x98BADCFEu, 0x10325476u, 0xC3D2E1F0u};
      for (uint32_t blk = 0; blk < max_blocks; blk++) {
        const uint32_t bs = blk_seq + blk, stage = bs % kH3Stages;
        if (MODE != 4) nbar_sync(bar0 + stage);
        if (MODE != 1 && MODE != 3 && blk < nblocks) sha1_chain80(&sm.wk[stage][lane][0], h);
        if (MODE != 4) nbar_arrive(bar0 + kH3Stages + stage);
      }
      if (have) digest_to_base32hex(h, out + 32 * (size_t)m);
    }
    chunk_seq += nchunks; blk_seq += max_blocks;
  }
}

}  // namespace kr
