// zk_seed.cuh — the randomness of a seeded call: every tape draw expanded on the device from the proof's 32-byte seed.
//
// The rule (normative statement in include/zkattest.h, restated in oracle/seed_tape.py):
//   stream(seed, domain, index) = ChaCha20 (RFC 8439 2.3, 20 rounds) keyed by the seed, nonce le32(domain) || le64(index),
//                                 blocks 0, 1, 2, ... concatenated
//   prover draw k            rnd(draw_modulus(k)) on stream(seed, 1, k): the first 32-byte big-endian candidate below
//                            the modulus (p256.n or p256.p = tom.order, a function of k alone)
//   verifier 32-byte slot t  the first 32-byte candidate of stream(seed, 2, t) below p256.n (GK drains, then exp drains)
//   verifier index byte i    rnd(S - i) on stream(seed, 3, i): one byte per candidate
// The tasks below write exactly the tape layouts of include/zkattest.h into library-owned, 16-byte aligned rows, so the
// pipeline behind them is the tape-mode pipeline unchanged.  Pure ALU work (add, xor, rotate): no multiplier.
#pragma once
#include "zk_verify.cuh"

namespace zk {

enum : uint32_t { SEED_DOM_PROVE = 1, SEED_DOM_VERIFY = 2, SEED_DOM_INDEX = 3 };

ZK_HD uint32_t chacha_rotl(uint32_t x, int n) {
#if defined(__CUDA_ARCH__)
  return __funnelshift_l(x, x, n);
#else
  return (x << n) | (x >> (32 - n));
#endif
}
ZK_HD void chacha_qr(uint32_t& a, uint32_t& b, uint32_t& c, uint32_t& d) {
  a += b; d ^= a; d = chacha_rotl(d, 16);
  c += d; b ^= c; b = chacha_rotl(b, 12);
  a += b; d ^= a; d = chacha_rotl(d, 8);
  c += d; b ^= c; b = chacha_rotl(b, 7);
}
// One ChaCha20 block (RFC 8439 2.3): ks[i] = keystream word i, i.e. keystream bytes 4i .. 4i+3 little-endian.
ZK_HD void chacha20_block(uint32_t* ks, const uint32_t* key, uint32_t counter, uint32_t n0, uint32_t n1, uint32_t n2) {
  uint32_t s[16] = {0x61707865u, 0x3320646eu, 0x79622d32u, 0x6b206574u, key[0], key[1], key[2], key[3],
                    key[4], key[5], key[6], key[7], counter, n0, n1, n2};
  uint32_t x[16];
#pragma unroll
  for (int i = 0; i < 16; i++) x[i] = s[i];
#pragma unroll
  for (int r = 0; r < 10; r++) {
    chacha_qr(x[0], x[4], x[8], x[12]);
    chacha_qr(x[1], x[5], x[9], x[13]);
    chacha_qr(x[2], x[6], x[10], x[14]);
    chacha_qr(x[3], x[7], x[11], x[15]);
    chacha_qr(x[0], x[5], x[10], x[15]);
    chacha_qr(x[1], x[6], x[11], x[12]);
    chacha_qr(x[2], x[7], x[8], x[13]);
    chacha_qr(x[3], x[4], x[9], x[14]);
  }
#pragma unroll
  for (int i = 0; i < 16; i++) ks[i] = x[i] + s[i];
}

// the seed as the ChaCha20 key: word i = le32(seed[4i .. 4i+3])
ZK_HD void seed_key(uint32_t* key, const uint8_t* seed) {
  if (aligned16(seed)) {
    ld8v(key, reinterpret_cast<const uint32_t*>(seed));
    return;
  }
#pragma unroll
  for (int i = 0; i < 8; i++)
    key[i] = (uint32_t)seed[4 * i] | ((uint32_t)seed[4 * i + 1] << 8) | ((uint32_t)seed[4 * i + 2] << 16) |
             ((uint32_t)seed[4 * i + 3] << 24);
}

// rnd(m) for a 32-byte modulus m (8 little-endian limbs, m >= 2^255 so that a candidate passes with probability > 1/2) on
// stream(key, domain, index): out = the kept candidate as 8 words in memory order (bytes 4w .. 4w+3 of the draw, i.e.
// the keystream words themselves), ready to be stored as the 32 tape bytes.
ZK_HD void seed_draw32(uint32_t* out, const uint32_t* key, uint32_t domain, uint64_t index, const uint32_t* m) {
  for (uint32_t blk = 0;; blk++) {
    uint32_t ks[16];
    chacha20_block(ks, key, blk, domain, (uint32_t)index, (uint32_t)(index >> 32));
#pragma unroll
    for (int h = 0; h < 2; h++) {
      uint32_t v[8];   // the candidate as limbs: limb 7 - w is big-endian bytes 4w .. 4w+3
#pragma unroll
      for (int w = 0; w < 8; w++) v[7 - w] = bswap32(ks[8 * h + w]);
      if (lt_n<8>(v, m)) {
#pragma unroll
        for (int w = 0; w < 8; w++) out[w] = ks[8 * h + w];
        return;
      }
    }
  }
}

// rnd(limit) for 1 < limit <= 256 on stream(key, SEED_DOM_INDEX, i): one byte per candidate
ZK_HD uint32_t seed_index_byte(const uint32_t* key, uint32_t i, uint32_t limit) {
  for (uint32_t blk = 0;; blk++) {
    uint32_t ks[16];
    chacha20_block(ks, key, blk, SEED_DOM_INDEX, i, 0u);
    for (int j = 0; j < 64; j++) {
      const uint32_t v = (ks[j >> 2] >> (8 * (j & 3))) & 0xffu;
      if (v < limit) return v;
    }
  }
}

// p256.n (order_n) or p256.p = tom.order as 8 little-endian limbs
ZK_HD void seed_modulus(uint32_t* m, bool order_n) {
  m[0] = order_n ? 0xfc632551u : 0xffffffffu;
  m[1] = order_n ? 0xf3b9cac2u : 0xffffffffu;
  m[2] = order_n ? 0xa7179e84u : 0xffffffffu;
  m[3] = order_n ? 0xbce6faadu : 0u;
  m[4] = order_n ? 0xffffffffu : 0u;
  m[5] = order_n ? 0xffffffffu : 0u;
  m[6] = order_n ? 0u : 1u;
  m[7] = 0xffffffffu;
}
// modulus of prover draw k (include/zkattest.h tape order): comS1.r and alpha_i, r_i mod p256.n, the rest mod tom.order
ZK_HD bool prove_draw_mod_n(int k, int S) {
  return k == DRAW_COMS1_R || (k >= DRAW_REP0 && k < draws_before_items(S) && ((k - DRAW_REP0) % DRAWS_PER_REP) < 2);
}

// Prover draws [d0, d0 + span) of every row: thread t = (row t / span, draw d0 + t % span), one 32-byte draw in two
// 16-byte stores.  With zcount set, row b stops at prove_draws(zcount[b], n_b, S), the last draw its proof reads; n_b is
// the depth of the row's own ring when ring_of is set (a ring-set call, n then being the largest depth), else n.
struct SeedProveTapeTask {
  const uint8_t* seeds;   // [B][32]
  uint8_t* tape;          // [B][tape_stride], 16-byte aligned rows
  size_t tape_stride;
  int S, n, d0, span;
  const uint32_t* zcount; // [B] or null
  const uint32_t *ring_of, *ring_depth;   // [B], [R] or null
  ZK_HD void operator()(int t) const {
    const int b = t / span, k = d0 + t % span;
    if (zcount && k >= prove_draws((int)zcount[b], ring_of ? (int)ring_depth[ring_of[b]] : n, S)) return;
    uint32_t key[8], m[8], w[8];
    seed_key(key, seeds + (size_t)b * 32);
    seed_modulus(m, prove_draw_mod_n(k, S));
    seed_draw32(w, key, SEED_DOM_PROVE, (uint64_t)k, m);
    st8v(reinterpret_cast<uint32_t*>(tape + (size_t)b * tape_stride + (size_t)32 * k), w);
  }
};

// The verifier layout of every row (zk_verify.cuh): thread t = (row, slot).  Slots [0, 2n + 1 + 25K) are the 32-byte
// draws in order (GK drains, then the packed exp drains behind the index area); the V_IDX_PAD / 16 slots after them
// write the index area 16 bytes at a time (index bytes i < S - 2, zero padding behind).  With ring_of set (a ring-set
// call) a row has the layout of its own ring's depth n_b <= n, and the slots beyond it are idle.
struct SeedVerifyTapeTask {
  const uint8_t* seeds;   // [B][32]
  uint8_t* tape;          // [B][tape_stride], 16-byte aligned rows
  size_t tape_stride;
  int n, S, K;
  const uint32_t *ring_of, *ring_depth;   // [B], [R] or null
  ZK_HD int slots() const { return 2 * n + 1 + 25 * K + V_IDX_PAD / 16; }
  ZK_HD void operator()(int t) const {
    const int b = t / slots(), s = t % slots();
    const int g = 2 * (ring_of ? (int)ring_depth[ring_of[b]] : n) + 1, draws = g + 25 * K;
    if (s >= draws + V_IDX_PAD / 16) return;
    uint32_t key[8], w[8];
    seed_key(key, seeds + (size_t)b * 32);
    uint8_t* row = tape + (size_t)b * tape_stride;
    if (s < draws) {
      uint32_t m[8];
      seed_modulus(m, true);
      seed_draw32(w, key, SEED_DOM_VERIFY, (uint64_t)s, m);
      st8v(reinterpret_cast<uint32_t*>(row + (s < g ? (size_t)32 * s : (size_t)32 * s + V_IDX_PAD)), w);
      return;
    }
    const int j = s - draws;
#pragma unroll
    for (int q = 0; q < 4; q++) w[q] = 0;
    for (int q = 0; q < 16; q++) {
      const int i = 16 * j + q;
      if (i < S - 2) w[q >> 2] |= seed_index_byte(key, (uint32_t)i, (uint32_t)(S - i)) << (8 * (q & 3));
    }
    st4(row + (size_t)32 * g + 16 * j, w);
  }
};

// ---- hedged seeds (include/zkattest.h, "Hedged seeds"; restated in tests/hedge_rule.py) ----------------------------
//   ring digest  SHA-256("ZKAttest/hedge/ring/v1" || le32(N) || le32(n) || leaf_0 || leaf_1 || ...), leaf k = SHA-256 of
//                the 32-byte big-endian entries [1024 k, 1024 k + 1024) of the ring reduced and padded to 2^n entries
//                (all 2^n of them when 2^n <= 1024)
//   row seed     SHA-256("ZKAttest/hedge/prove/v1" || params digest || ring digest || seed (or 32 zero bytes) ||
//                msg_hash || sig || pk || le32(which))
// The seed of a row then feeds SeedProveTapeTask unchanged.
enum : int { HEDGE_LEAF_BITS = 10 };

ZK_HD void sha_tag(Sha256& h, const char* s) {
  while (*s) h.put((uint8_t)*s++);
}
// the digest as its 32 bytes in memory order (16-byte aligned destination)
ZK_HD void sha_store(Sha256& h, uint8_t* out) {
  uint32_t d[8];
  h.final256(d);
#pragma unroll
  for (int i = 0; i < 8; i++) d[i] = bswap32(d[i]);
  st8v(reinterpret_cast<uint32_t*>(out), d);
}
ZK_HD uint32_t hedge_leaves(int n) { return n > HEDGE_LEAF_BITS ? 1u << (n - HEDGE_LEAF_BITS) : 1u; }

// The ring digest of R rings, two launches: leaf (thread = one leaf of one ring) then root (thread = one ring).  The
// entries are read from the prepared rings (RingPrepTask / RingSetPrepTask: reduced, padded, Montgomery form), so the
// digest covers exactly the ring the proof is made against.  One ring: ring_base / ring_size / ring_depth / leaf_off
// null, R = 1, size N and depth n.
struct RingDigestTask {
  const uint32_t* ring_m;      // [entries][8]
  const uint32_t *ring_base, *ring_size, *ring_depth, *leaf_off;   // [R], [R], [R], [R + 1] or null
  uint32_t N, n, R;
  uint8_t* leaves;             // [total leaves][32]
  uint8_t* digest;             // [R][32]
  bool root;
  ZK_HD void operator()(int t) const {
    if (root) {
      const uint32_t r = (uint32_t)t, d = ring_depth ? ring_depth[r] : n;
      const uint8_t* lv = leaves + (size_t)32 * (leaf_off ? leaf_off[r] : 0u);
      Sha256 h;
      h.init();
      sha_tag(h, "ZKAttest/hedge/ring/v1");
      h.put4(ring_size ? ring_size[r] : N);
      h.put4(d);
      for (uint32_t k = 0; k < hedge_leaves((int)d); k++) h.update(lv + (size_t)32 * k, 32);
      sha_store(h, digest + (size_t)32 * r);
      return;
    }
    uint32_t r = 0;
    if (leaf_off) {   // the last ring whose first leaf is <= t
      uint32_t lo = 0, hi = R - 1;
      while (lo < hi) {
        const uint32_t mid = (lo + hi + 1) >> 1;
        if (leaf_off[mid] <= (uint32_t)t) lo = mid; else hi = mid - 1;
      }
      r = lo;
    }
    const uint32_t d = ring_depth ? ring_depth[r] : n;
    const uint32_t k = (uint32_t)t - (leaf_off ? leaf_off[r] : 0u);
    const uint32_t count = d > HEDGE_LEAF_BITS ? 1u << HEDGE_LEAF_BITS : 1u << d;
    const uint32_t* e = ring_m + (size_t)8 * ((ring_base ? ring_base[r] : 0u) + (k << HEDGE_LEAF_BITS));
    Sha256 h;
    h.init();
    for (uint32_t j = 0; j < count; j++) {
      uint32_t m[8], v[8];
      ld<8>(m, e + (size_t)8 * j);
      Tomq::from_mont(v, m);
#pragma unroll
      for (int w = 7; w >= 0; w--) h.put4(bswap32(v[w]));   // big-endian: the most significant limb first
    }
    sha_store(h, leaves + (size_t)32 * t);
  }
};

// One thread per row: the row's hedged seed into out[b] (16-byte aligned rows of 32 bytes).  ring_of null: one ring.
struct SeedHedgeTask {
  uint32_t params_digest[8];   // the 32 bytes of zka_params' digest as little-endian words
  const uint8_t* ring_digest;  // [R][32]
  const uint32_t* ring_of;     // [B] or null
  const uint8_t *seeds, *msg_hash, *sig, *pk;   // seeds may be null (32 zero bytes)
  const uint32_t* which;
  uint8_t* out;                // [B][32]
  ZK_HD void operator()(int b) const {
    Sha256 h;
    h.init();
    sha_tag(h, "ZKAttest/hedge/prove/v1");
#pragma unroll
    for (int i = 0; i < 8; i++) h.put4(params_digest[i]);
    h.update(ring_digest + (size_t)32 * (ring_of ? ring_of[b] : 0u), 32);
    if (seeds) {
      h.update(seeds + (size_t)32 * b, 32);
    } else {
#pragma unroll
      for (int i = 0; i < 8; i++) h.put4(0u);
    }
    h.update(msg_hash + (size_t)32 * b, 32);
    h.update(sig + (size_t)64 * b, 64);
    h.update(pk + (size_t)65 * b, 65);
    h.put4(which[b]);
    sha_store(h, out + (size_t)32 * b);
  }
};

}  // namespace zk
