// zk_sha256.cuh — SHA-256 for the Fiat-Shamir challenges.
//
// Replaces WebCrypto `crypto.subtle.digest('SHA-256', bytes)` inside hashPoints
// (/root/reference/src/curves/group.ts:221-233).  The message is the concatenation of
// 65/67-byte point encodings gathered from several places, so the hasher is streaming:
// update() with arbitrary byte spans, final80() returns the first 10 digest bytes as the
// 80-bit challenge (two words: hi 16 bits, lo 64 bits).
#pragma once
#include "zk_field.cuh"

namespace zk {

struct ShaH { uint32_t v[8]; };
struct ShaW { uint32_t v[16]; };

ZK_HD uint32_t sha_rotr(uint32_t x, int n) { return (x >> n) | (x << (32 - n)); }

// One compression.  On the device this is ONE non-inlined function with register-passed state: the
// streaming hasher calls it from a dozen places, and inlined copies (2 000 instructions each) made the
// hash kernels ~900 KB of code that a single resident warp per SM fetched from L2 over and over.
ZK_HD ShaH sha256_compress_body(ShaH hs, const ShaW& ws) {
  constexpr uint32_t k[64] = {
      0x428a2f98, 0x71374491, 0xb5c0fbcf, 0xe9b5dba5, 0x3956c25b, 0x59f111f1, 0x923f82a4, 0xab1c5ed5,
      0xd807aa98, 0x12835b01, 0x243185be, 0x550c7dc3, 0x72be5d74, 0x80deb1fe, 0x9bdc06a7, 0xc19bf174,
      0xe49b69c1, 0xefbe4786, 0x0fc19dc6, 0x240ca1cc, 0x2de92c6f, 0x4a7484aa, 0x5cb0a9dc, 0x76f988da,
      0x983e5152, 0xa831c66d, 0xb00327c8, 0xbf597fc7, 0xc6e00bf3, 0xd5a79147, 0x06ca6351, 0x14292967,
      0x27b70a85, 0x2e1b2138, 0x4d2c6dfc, 0x53380d13, 0x650a7354, 0x766a0abb, 0x81c2c92e, 0x92722c85,
      0xa2bfe8a1, 0xa81a664b, 0xc24b8b70, 0xc76c51a3, 0xd192e819, 0xd6990624, 0xf40e3585, 0x106aa070,
      0x19a4c116, 0x1e376c08, 0x2748774c, 0x34b0bcb5, 0x391c0cb3, 0x4ed8aa4a, 0x5b9cca4f, 0x682e6ff3,
      0x748f82ee, 0x78a5636f, 0x84c87814, 0x8cc70208, 0x90befffa, 0xa4506ceb, 0xbef9a3f7, 0xc67178f2};
  uint32_t a = hs.v[0], b = hs.v[1], c = hs.v[2], d = hs.v[3], e = hs.v[4], f = hs.v[5], g = hs.v[6], hh = hs.v[7];
  uint32_t m[16];
#pragma unroll
  for (int i = 0; i < 16; i++) m[i] = ws.v[i];
#pragma unroll
  for (int i = 0; i < 64; i++) {
    uint32_t wi;
    if (i < 16) {
      wi = m[i];
    } else {
      uint32_t w15 = m[(i + 1) & 15], w2 = m[(i + 14) & 15];
      uint32_t s0 = sha_rotr(w15, 7) ^ sha_rotr(w15, 18) ^ (w15 >> 3);
      uint32_t s1 = sha_rotr(w2, 17) ^ sha_rotr(w2, 19) ^ (w2 >> 10);
      wi = m[i & 15] + s0 + m[(i + 9) & 15] + s1;
      m[i & 15] = wi;
    }
    uint32_t S1 = sha_rotr(e, 6) ^ sha_rotr(e, 11) ^ sha_rotr(e, 25);
    uint32_t ch = (e & f) ^ (~e & g);
    uint32_t t1 = hh + S1 + ch + k[i] + wi;
    uint32_t S0 = sha_rotr(a, 2) ^ sha_rotr(a, 13) ^ sha_rotr(a, 22);
    uint32_t mj = (a & b) ^ (a & c) ^ (b & c);
    uint32_t t2 = S0 + mj;
    hh = g; g = f; f = e; e = d + t1; d = c; c = b; b = a; a = t1 + t2;
  }
  hs.v[0] += a; hs.v[1] += b; hs.v[2] += c; hs.v[3] += d; hs.v[4] += e; hs.v[5] += f; hs.v[6] += g; hs.v[7] += hh;
  return hs;
}
#if defined(__CUDACC__)
static __device__ __noinline__ ShaH sha256_compress_fn(ShaH hs, ShaW ws) { return sha256_compress_body(hs, ws); }
#endif

struct Sha256 {
  uint32_t h[8];
  uint32_t w[16];   // current block, big-endian words
  uint32_t fill;    // bytes in current block
  uint64_t total;   // total bytes

  ZK_HD void init() {
    h[0] = 0x6a09e667; h[1] = 0xbb67ae85; h[2] = 0x3c6ef372; h[3] = 0xa54ff53a;
    h[4] = 0x510e527f; h[5] = 0x9b05688c; h[6] = 0x1f83d9ab; h[7] = 0x5be0cd19;
#pragma unroll
    for (int i = 0; i < 16; i++) w[i] = 0;
    fill = 0;
    total = 0;
    cur = 0;
  }

  ZK_HD void compress() {
    ShaH hs;
    ShaW ws;
#pragma unroll
    for (int i = 0; i < 8; i++) hs.v[i] = h[i];
#pragma unroll
    for (int i = 0; i < 16; i++) ws.v[i] = w[i];
#if defined(__CUDA_ARCH__)
    hs = sha256_compress_fn(hs, ws);
#else
    hs = sha256_compress_body(hs, ws);
#endif
#pragma unroll
    for (int i = 0; i < 8; i++) h[i] = hs.v[i];
    fill -= 64;   // bytes still pending in `cur` (0..3) belong to the next block
  }

  // The block buffer is a 16-word FIFO with static indices only (w[15] is the newest word), so it
  // stays in registers; `fill` counts bytes of the current block, `cur` gathers 4 bytes.
  uint32_t cur;
  ZK_HD void push_word(uint32_t v) {
#pragma unroll
    for (int i = 0; i < 15; i++) w[i] = w[i + 1];
    w[15] = v;
  }
  ZK_HD void put(uint8_t byte) {
    cur = (cur << 8) | byte;
    fill++;
    total++;
    if ((fill & 3) == 0) {
      push_word(cur);
      if (fill == 64) compress();
    }
  }
  // four stream bytes at once, given as the little-endian word loaded from memory
  ZK_HD void put4(uint32_t lw) {
    const uint32_t bw = (lw << 24) | ((lw & 0xff00u) << 8) | ((lw >> 8) & 0xff00u) | (lw >> 24);
    const int nb = (int)(fill & 3);                       // bytes pending in `cur`
    const uint64_t v = ((uint64_t)cur << 32) | bw;
    push_word((uint32_t)(v >> (8 * nb)));
    cur = bw;                                             // its low nb bytes are the new pending bytes
    fill += 4;
    total += 4;
    if (fill >= 64) compress();
  }
  // Spans are consumed in groups of 16 aligned words; the loads of the NEXT group are issued before the
  // current group is hashed, so a thread waits for memory once per span instead of once per word
  // (one thread hashes up to 16 KB alone: exp.ts:184-190).
  ZK_HD void update(const uint8_t* p, int n) {
    int i = 0;
    while (i < n && (((size_t)(p + i)) & 3)) put(p[i++]);
    const uint32_t* q = reinterpret_cast<const uint32_t*>(p + i);
    int nw = (n - i) >> 2;
    i += 4 * nw;
    uint32_t a[16], b[16];
#pragma unroll
    for (int j = 0; j < 16; j++) a[j] = j < nw ? q[j] : 0u;
    while (nw > 0) {
      const int m = nw < 16 ? nw : 16;
#pragma unroll
      for (int j = 0; j < 16; j++) b[j] = 16 + j < nw ? q[16 + j] : 0u;
#pragma unroll
      for (int j = 0; j < 16; j++)
        if (j < m) put4(a[j]);
#pragma unroll
      for (int j = 0; j < 16; j++) a[j] = b[j];
      q += 16;
      nw -= m;
    }
    for (; i < n; i++) put(p[i]);
  }
  // one encoded point (64 <= n <= 68 bytes) already loaded as 17 little-endian words
  ZK_HD void feed17(const uint32_t* t, int n) {
    const int nf = n >> 2;
#pragma unroll
    for (int j = 0; j < 17; j++)
      if (j < nf) put4(t[j]);
    for (int k = 0; k < (n & 3); k++) put((uint8_t)(t[16] >> (8 * k)));   // n in [64,68): the tail lives in t[16]
  }
  ZK_HD void pad() {
    const uint64_t bits = total * 8;
    put(0x80);
    while ((fill & 3) != 0) put(0);
    // now `fill` is a multiple of 4; pad with zero words up to byte 56, then the length
    if (fill > 56) {
      while (fill != 0) { push_word(0); fill += 4; if (fill == 64) compress(); }
    }
    while (fill != 56) { push_word(0); fill += 4; }
    push_word((uint32_t)(bits >> 32));
    push_word((uint32_t)bits);
    compress();
  }
  // the whole digest as eight big-endian words
  ZK_HD void final256(uint32_t* d8) {
    pad();
#pragma unroll
    for (int i = 0; i < 8; i++) d8[i] = h[i];
  }
  // digest[0..9] as (hi16, lo64): challenge = hi16 * 2^64 + lo64
  ZK_HD void final80(uint32_t* c3) {  // c3[0] = low 32, c3[1] = mid 32, c3[2] = top 16 bits
    pad();
    // digest bytes 0..9 = h0 (4) h1 (4) top half of h2 (2)  -> 80-bit big-endian integer
    uint32_t top16 = h[0] >> 16;
    uint32_t mid = (h[0] << 16) | (h[1] >> 16);
    uint32_t low = (h[1] << 16) | (h[2] >> 16);
    c3[0] = low;
    c3[1] = mid;
    c3[2] = top16;
  }
};

}  // namespace zk
