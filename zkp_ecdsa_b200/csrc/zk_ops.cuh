// zk_ops.cuh — building-block tasks: precomputed tables, scalar multiplication, batched
// affine normalisation + serialisation, SHA-256 over point encodings.
//
// A "task" is a functor `void operator()(int t) const` executed once per work item; the
// CUDA build runs it as one thread of a grid (zk_launch.cuh).  All tables and staging
// buffers live in HBM/L2: the path is integer-pipe bound (SURVEY.md 8(d)), the staging
// traffic is < 1 % of HBM bandwidth.
//
// Reference mapping:
//   Point.mul / Point.dblmul (4-bit windows, /root/reference/src/curves/group.ts:97-152)
//     -> positional fixed-window tables, NO doublings at evaluation time:
//        k*P = sum_j T[j][digit_j(k)],  T[j][d] = d * 2^(w j) * P   (affine / precomputed)
//   toAffine + toBytes (weier.ts:231-255, edwards.ts:184-203; one invEuclid each)
//     -> Montgomery's trick over chunks of points, one Fermat inversion per chunk.
#pragma once
#include "zk_curves.cuh"
#include "zk_layout.h"
#include "zk_sha256.cuh"

namespace zk {

#if defined(__CUDA_ARCH__)
#define ZK_SET_STATUS(ptr, code) atomicCAS((int*)(ptr), 0, (int)(code))
// the smallest key wins, whichever thread or kernel posts it first (the verifier's exp-side status keys, zk_verify.cuh)
#define ZK_POST_MIN(ptr, key) atomicMin((int*)(ptr), (int)(key))
// first error wins, except that `code` also replaces the later-stage error `over` (used when the two
// stages run side by side in one grid: the outcome equals running this stage first)
#define ZK_SET_STATUS_OVER(ptr, code, over) \
  do {                                      \
    atomicCAS((int*)(ptr), 0, (int)(code)); \
    atomicCAS((int*)(ptr), (int)(over), (int)(code)); \
  } while (0)
#else
#define ZK_SET_STATUS_OVER(ptr, code, over)              \
  do {                                                   \
    if (*(ptr) == 0 || *(ptr) == (over)) *(ptr) = (code); \
  } while (0)
#define ZK_SET_STATUS(ptr, code) \
  do {                           \
    if (*(ptr) == 0) *(ptr) = (code); \
  } while (0)
#define ZK_POST_MIN(ptr, key)             \
  do {                                    \
    if ((int)(key) < *(ptr)) *(ptr) = (int)(key); \
  } while (0)
#endif

// ----------------------------------------------------------------------------- loads/stores
template <int N>
ZK_HD void ld(uint32_t* r, const uint32_t* p) {
#pragma unroll
  for (int i = 0; i < N; i++) r[i] = p[i];
}
template <int N>
ZK_HD void st(uint32_t* p, const uint32_t* r) {
#pragma unroll
  for (int i = 0; i < N; i++) p[i] = r[i];
}

enum : int {
  P256_PROJ_WORDS = 24,
  P256_AFF_WORDS = 16,
#if defined(ZKA_PG_WAR256)
  TOM_PROJ_WORDS = 24,   // war256 build: homogeneous (X, Y, Z), 8 limbs each
  TOM_E2_WORDS = 24,     // a commitment for the normaliser: (X, Y, Z) as well
  TOM_AFF_WORDS = 16,    // affine (x, y), Montgomery
  TOM_PRE_WORDS = 16,    // table entry / parsed point = affine (x, y): one 64-byte half line
#else
  TOM_PROJ_WORDS = 28,   // X, Y, Z (T is not needed after the last addition) + 1 pad word: 7 x 16 bytes
  TOM_E2_WORDS = 36,     // a commitment for the normaliser: E, F, G, H of its last addition (tom2_madd_end), 9 x 16 bytes
  TOM_AFF_WORDS = 18,    // x', y on the a'=1 image curve, Montgomery
  TOM_PRE_WORDS = 32,    // x', y, k = d' x' y + 5 pad words: one 128-byte line per entry
#endif
  NORM_CHUNK_MAX = 64,   // max points per Montgomery-trick chunk (one Fermat inversion each)
};


#if defined(ZKA_PG_WAR256)
// staged war256 points: X, Y, Z at words 0, 8, 16 of a 96-byte slot; table entries are affine pairs
ZK_HD void tom_st_xyz(uint32_t* m, const uint32_t* x, const uint32_t* y, const uint32_t* z) {
  st<8>(m, x); st<8>(m + 8, y); st<8>(m + 16, z);
}
ZK_HD void tom_ld_xyz(uint32_t* x, uint32_t* y, uint32_t* z, const uint32_t* m) {
  ld<8>(x, m); ld<8>(y, m + 8); ld<8>(z, m + 16);
}
ZK_HD void tom_ld_pre(TomPre& q, const uint32_t* m) { ld<8>(q.x, m); ld<8>(q.y, m + 8); }
#else
// staged tomEdwards256 points (X, Y, Z at words 0, 9, 18 of a 112-byte, 16-byte aligned slot):
// seven 16-byte transactions instead of 27 four-byte ones (the slots are strided per thread)
ZK_HD void tom_st_xyz(uint32_t* m, const uint32_t* x, const uint32_t* y, const uint32_t* z) {
  uint32_t w[28];
#pragma unroll
  for (int i = 0; i < 9; i++) { w[i] = x[i]; w[9 + i] = y[i]; w[18 + i] = z[i]; }
  w[27] = 0;
#if defined(__CUDA_ARCH__)
  uint4* v = reinterpret_cast<uint4*>(m);
#pragma unroll
  for (int i = 0; i < 7; i++) v[i] = make_uint4(w[4 * i], w[4 * i + 1], w[4 * i + 2], w[4 * i + 3]);
#else
  for (int i = 0; i < 28; i++) m[i] = w[i];
#endif
}
ZK_HD void tom_ld_xyz(uint32_t* x, uint32_t* y, uint32_t* z, const uint32_t* m) {
  uint32_t w[28];
#if defined(__CUDA_ARCH__)
  const uint4* v = reinterpret_cast<const uint4*>(m);
#pragma unroll
  for (int i = 0; i < 7; i++) {
    const uint4 u = v[i];
    w[4 * i] = u.x; w[4 * i + 1] = u.y; w[4 * i + 2] = u.z; w[4 * i + 3] = u.w;
  }
#else
  for (int i = 0; i < 28; i++) w[i] = m[i];
#endif
#pragma unroll
  for (int i = 0; i < 9; i++) { x[i] = w[i]; y[i] = w[9 + i]; z[i] = w[18 + i]; }
}
// staged E2 commitments for the normaliser (E, F, G, H at words 0, 9, 18, 27 of a 144-byte slot): nine 16-byte transactions
ZK_HD void tom_st_efgh(uint32_t* m, const TomEfgh& p) {
  uint32_t w[36];
#pragma unroll
  for (int i = 0; i < 9; i++) { w[i] = p.e[i]; w[9 + i] = p.f[i]; w[18 + i] = p.g[i]; w[27 + i] = p.h[i]; }
#if defined(__CUDA_ARCH__)
  uint4* v = reinterpret_cast<uint4*>(m);
#pragma unroll
  for (int i = 0; i < 9; i++) v[i] = make_uint4(w[4 * i], w[4 * i + 1], w[4 * i + 2], w[4 * i + 3]);
#else
  for (int i = 0; i < 36; i++) m[i] = w[i];
#endif
}
ZK_HD void tom_ld_efgh(uint32_t* e, uint32_t* f, uint32_t* g, uint32_t* h, const uint32_t* m) {
  uint32_t w[36];
#if defined(__CUDA_ARCH__)
  const uint4* v = reinterpret_cast<const uint4*>(m);
#pragma unroll
  for (int i = 0; i < 9; i++) {
    const uint4 u = v[i];
    w[4 * i] = u.x; w[4 * i + 1] = u.y; w[4 * i + 2] = u.z; w[4 * i + 3] = u.w;
  }
#else
  for (int i = 0; i < 36; i++) w[i] = m[i];
#endif
#pragma unroll
  for (int i = 0; i < 9; i++) { e[i] = w[i]; f[i] = w[9 + i]; g[i] = w[18 + i]; h[i] = w[27 + i]; }
}

// negate a table entry of the a = -1 image curve: -(w, v) = (-w, v) swaps v - w and v + w and negates 2 d2 w v
ZK_HD void tom2_pre_neg(TomPre& q, bool neg) {
  uint32_t nk[9];
  Tomp::neg(nk, q.k);
#pragma unroll
  for (int i = 0; i < 9; i++) {
    const uint32_t a = q.x[i], b = q.y[i];
    q.x[i] = neg ? b : a;
    q.y[i] = neg ? a : b;
    q.k[i] = neg ? nk[i] : q.k[i];
  }
}
ZK_HD void tom_ld_pre(TomPre& q, const uint32_t* m) {
#if defined(__CUDA_ARCH__)
  // one 128-byte line, eight 16-byte loads (entries are 128-byte aligned)
  const uint4* v = reinterpret_cast<const uint4*>(m);
  uint32_t w[32];
#pragma unroll
  for (int i = 0; i < 7; i++) {
    uint4 u = __ldg(v + i);
    w[4 * i] = u.x; w[4 * i + 1] = u.y; w[4 * i + 2] = u.z; w[4 * i + 3] = u.w;
  }
#pragma unroll
  for (int i = 0; i < 9; i++) { q.x[i] = w[i]; q.y[i] = w[9 + i]; q.k[i] = w[18 + i]; }
#else
  ld<9>(q.x, m); ld<9>(q.y, m + 9); ld<9>(q.k, m + 18);
#endif
}

#endif

// 16-byte vector loads and stores of the device build; the host simulator moves the same words one at a time
ZK_HD void ld4(uint32_t* w, const void* p) {
#if defined(__CUDA_ARCH__)
  const uint4 u = *reinterpret_cast<const uint4*>(p);
  w[0] = u.x; w[1] = u.y; w[2] = u.z; w[3] = u.w;
#else
  const uint32_t* q = reinterpret_cast<const uint32_t*>(p);
  for (int i = 0; i < 4; i++) w[i] = q[i];
#endif
}
ZK_HD void st4(void* p, const uint32_t* w) {
#if defined(__CUDA_ARCH__)
  *reinterpret_cast<uint4*>(p) = make_uint4(w[0], w[1], w[2], w[3]);
#else
  uint32_t* q = reinterpret_cast<uint32_t*>(p);
  for (int i = 0; i < 4; i++) q[i] = w[i];
#endif
}
// a 32-byte row of 8 words (scalar rows, affine coordinates; every such buffer is 16-byte aligned): two 16-byte transactions
ZK_HD void ld8v(uint32_t* r, const uint32_t* p) { ld4(r, p); ld4(r + 4, p + 4); }
ZK_HD void st8v(uint32_t* p, const uint32_t* r) { st4(p, r); st4(p + 4, r + 4); }
ZK_HD bool aligned16(const void* p) { return ((size_t)p & 15) == 0; }

// Encoded point (tag || x || y, big-endian coordinates of CB bytes) written into a BSTRIDE slot: five 16-byte stores
// into a 16-byte aligned slot (every staging slot), 20 word stores into any other 4-byte aligned one.  The byte index
// of every output position is a compile-time constant after unrolling; bytes past the encoding are written as 0.
template <int N, int CB>
ZK_HD uint32_t enc_byte(int i, uint32_t tag, const uint32_t* x, const uint32_t* y) {
  if (i == 0) return tag;
  if (i >= 1 + 2 * CB) return 0u;
  const uint32_t* c = i <= CB ? x : y;
  const int pos = CB - 1 - (i <= CB ? i - 1 : i - 1 - CB);   // byte significance
  return (pos >> 2) < N ? ((c[pos >> 2] >> (8 * (pos & 3))) & 0xffu) : 0u;
}
template <int N, int CB>
ZK_HD void store_point_words(uint8_t* o, uint32_t tag, const uint32_t* x, const uint32_t* y) {
  uint32_t w[BSTRIDE / 4];
#pragma unroll
  for (int j = 0; j < BSTRIDE / 4; j++)
    w[j] = enc_byte<N, CB>(4 * j, tag, x, y) | (enc_byte<N, CB>(4 * j + 1, tag, x, y) << 8) |
           (enc_byte<N, CB>(4 * j + 2, tag, x, y) << 16) | (enc_byte<N, CB>(4 * j + 3, tag, x, y) << 24);
  if (aligned16(o)) {
#pragma unroll
    for (int j = 0; j < BSTRIDE / 16; j++) st4(o + 16 * j, w + 4 * j);
  } else {
    uint32_t* ow = reinterpret_cast<uint32_t*>(o);
#pragma unroll
    for (int j = 0; j < BSTRIDE / 4; j++) ow[j] = w[j];
  }
}

// digit j of width w (w in {4, 8}) of a canonical 256-bit scalar
ZK_HD uint32_t digit4(const uint32_t* k, int j) { return (k[j >> 3] >> (4 * (j & 7))) & 15u; }
ZK_HD uint32_t digit8(const uint32_t* k, int j) { return (k[j >> 2] >> (8 * (j & 3))) & 255u; }
// generic: bits [pos, pos+w) of a 256-bit scalar, w <= 24
ZK_HD uint32_t digit_w(const uint32_t* k, int pos, int w) {
  int wi = pos >> 5, sh = pos & 31;
  uint64_t v = k[wi];
  if (wi + 1 < 8) v |= (uint64_t)k[wi + 1] << 32;
  return (uint32_t)(v >> sh) & ((1u << w) - 1u);
}

// Fixed-base tables hold SIGNED digits: k = sum_j d_j 2^(w j), d_j in [-2^(w-1), 2^(w-1)], so a window stores the
// multiples 0 .. 2^(w-1) only (half the memory of unsigned digits at the same number of lookups); a negative
// digit negates the entry on the fly.  ceil(257 / w) windows: the carry out of the top data window needs one
// more window only when w divides 256.
ZK_HD int fb_entries(int w) { return (1 << (w - 1)) + 1; }
ZK_HD int fb_windows(int w) { return (256 + w) / w; }
// digit j of k in signed form: returns |d_j| and its sign; `carry` is the running carry (start with 0)
// the w-bit digit at bit `pos`
ZK_HD uint32_t signed_digit_at(const uint32_t* k, int pos, int w, uint32_t& carry, bool& neg) {
  uint32_t d = carry;
  if (pos < 256) d += digit_w(k, pos, (256 - pos) < w ? (256 - pos) : w);
  const uint32_t half = 1u << (w - 1);
  neg = d > half;
  carry = neg ? 1u : 0u;
  return neg ? (1u << w) - d : d;
}
ZK_HD uint32_t signed_digit(const uint32_t* k, int j, int w, uint32_t& carry, bool& neg) {
  return signed_digit_at(k, j * w, w, carry, neg);
}

// Shape of a positional signed-digit table whose windows are not all equally wide: the first n_lo of its nwin windows
// have w bits, the others w + 1.  With one width the 257 bits of a walk (256 of the scalar and the recoding's carry)
// take 12 windows at w = 22 and at w = 23, and 11 only at w = 24; seven windows of 23 bits and four of 24 cover exactly
// 257 bits in 11 lookups with a third less memory than 11 x 24.  The wide windows are the top ones, so bit position and
// entry offset of window j stay one multiply-add and one shift.  A uniform table is the case n_lo = nwin.
struct FbShape {
  int w, nwin, n_lo;
  ZK_HD int wide(int j) const { return j > n_lo ? j - n_lo : 0; }   // wide windows below window j
  ZK_HD int width(int j) const { return w + (j >= n_lo ? 1 : 0); }
  ZK_HD int bitpos(int j) const { return j * w + wide(j); }
  ZK_HD int bits() const { return bitpos(nwin); }
  ZK_HD size_t entries(int j) const { return ((size_t)1 << (width(j) - 1)) + 1; }
  ZK_HD size_t offset(int j) const { return (size_t)j * (size_t)fb_entries(w) + ((size_t)wide(j) << (w - 1)); }   // entries below window j
  ZK_HD size_t total() const { return offset(nwin); }
};
ZK_HD FbShape fb_uniform(int w) { return FbShape{w, fb_windows(w), fb_windows(w)}; }
// the shape that covers exactly 257 bits in nwin lookups (nwin < 257): w = floor(257 / nwin), 257 - w nwin wide windows
ZK_HD FbShape fb_lookups(int nwin) {
  const int w = 257 / nwin;
  return FbShape{w, nwin, nwin - (257 - w * nwin)};
}
// digit j of k on a table of shape s, otherwise as above
ZK_HD uint32_t signed_digit(const uint32_t* k, int j, const FbShape& s, uint32_t& carry, bool& neg) {
  return signed_digit_at(k, s.bitpos(j), s.width(j), carry, neg);
}

// read a 32-byte big-endian tape draw into 8 limbs.  A 16-byte aligned draw (every row of the library's own tape
// buffers, and device tapes whose base and stride are multiples of 16) is two read-only 16-byte loads and eight
// byte swaps; any other address takes 32 single-byte loads, so every caller pointer and stride stays legal.  The
// buffer must not be written by the same kernel (the 16-byte loads go through the non-coherent read-only path).
ZK_HD uint32_t bswap32(uint32_t x) {
#if defined(__CUDA_ARCH__)
  return __byte_perm(x, 0u, 0x0123);
#else
  return (x >> 24) | ((x >> 8) & 0xff00u) | ((x << 8) & 0xff0000u) | (x << 24);
#endif
}
ZK_HD void tape_draw(uint32_t* r, const uint8_t* tape, int draw) {
  const uint8_t* p = tape + 32 * (size_t)draw;
#if defined(__CUDA_ARCH__)
  if (aligned16(p)) {
    const uint4 a = __ldg(reinterpret_cast<const uint4*>(p)), b = __ldg(reinterpret_cast<const uint4*>(p) + 1);
    // stream word w (bytes 4w..4w+3, most significant first) is limb 7 - w
    r[7] = bswap32(a.x); r[6] = bswap32(a.y); r[5] = bswap32(a.z); r[4] = bswap32(a.w);
    r[3] = bswap32(b.x); r[2] = bswap32(b.y); r[1] = bswap32(b.z); r[0] = bswap32(b.w);
    return;
  }
#endif
#pragma unroll
  for (int i = 0; i < 8; i++) {
    const uint8_t* q = p + 28 - 4 * i;
    r[i] = ((uint32_t)q[0] << 24) | ((uint32_t)q[1] << 16) | ((uint32_t)q[2] << 8) | (uint32_t)q[3];
  }
}

// ============================================================================ P-256 tables
#define WEI_PT P256Pt
#define WEI_AFF P256Aff
#define WEI_JAC P256Jac
#define WEI_F P256p
#define WEI_FN(n) p256_##n
#define WEI_T(n) P256##n
#include "zk_weier_ops.inc"
#undef WEI_PT
#undef WEI_AFF
#undef WEI_JAC
#undef WEI_F
#undef WEI_FN
#undef WEI_T

// ---- per-KEY tables of the prover: the generic signed-digit format [fb_windows(w)][fb_entries(w)][16] with the window
// bits chosen ON THE DEVICE from the number of distinct keys of the chunk (KeyRankTask).  Grids and buffers are sized
// for the worst case (every proof its own key, w = 5: KEY_CAP entries per proof); fewer keys get wider windows inside
// the same memory: 256 keys in a chunk of 4096 proofs -> w = 8, 33 instead of 52 lookups per alpha*pk.
enum : int { KEY_W_MIN = 5, KEY_W_MAX = 8, KEY_CAP = 52 * 17 };
ZK_HD int key_window_bits(uint32_t count, uint32_t B, uint32_t uses) {   // uses = products per proof (S + 2)
  int best = KEY_W_MIN;
  uint64_t best_cost = ~0ull;
  for (int w = KEY_W_MIN; w <= KEY_W_MAX; w++) {
    const uint64_t nwin = (uint64_t)fb_windows(w), ne = (uint64_t)fb_entries(w);
    if (w > KEY_W_MIN && (uint64_t)count * nwin * ne > (uint64_t)B * KEY_CAP) break;
    // building an entry = one addition + its share of a normalisation (~2 mixed additions), used `uses` times per proof
    const uint64_t cost = nwin * ((uint64_t)count * (ne - 1) * 2 + (uint64_t)B * uses);
    if (cost < best_cost) { best_cost = cost; best = w; }
  }
  return best;
}
ZK_HD size_t key_table_words(int w) { return (size_t)fb_windows(w) * fb_entries(w) * P256_AFF_WORDS; }

// Per-base SIGNED 5-bit table (the per-proof table of R): k = sum_j d_j 32^j with d_j in [-16, 16],
// 52 windows x 16 entries (1..16 multiples); a negative digit negates y of the affine entry.
// 52 mixed additions per scalar multiplication instead of 64 with unsigned 4-bit windows, and the
// table is smaller (832 entries instead of 960).
enum : int { RT_W = 5, RT_NWIN = 52, RT_ROW = 16, RT_ENTRIES = RT_NWIN * RT_ROW };
struct P256RowsSignedTask {
  const uint32_t* pows;  // [nbase*RT_NWIN][24]
  uint32_t* rows;        // [nbase*RT_NWIN][RT_ROW][24]: entry d-1 = d * pows
  const uint32_t* count_dev = nullptr;   // optional: number of bases actually present
  ZK_HD void operator()(int t) const {
    if (count_dev && (uint32_t)(t / RT_NWIN) >= *count_dev) return;
    P256Pt p, acc;
    p256_ld_proj(p, pows + (size_t)t * P256_PROJ_WORDS);
    acc = p;
    uint32_t* out = rows + (size_t)t * RT_ROW * P256_PROJ_WORDS;
    for (int d = 1; d <= RT_ROW; d++) {
      p256_st_proj(out + (size_t)(d - 1) * P256_PROJ_WORDS, acc);
      if (d < RT_ROW) p256_add(acc, acc, p);
    }
  }
};
// acc += k * base on the signed 5-bit per-base table [RT_NWIN][RT_ROW] (P256RowsSignedTask)
ZK_HD void p256_accum_rtab(P256Pt& acc, const uint32_t* tab, const uint32_t* k) {
  uint32_t carry = 0;
  for (int j = 0; j < RT_NWIN; j++) {
    const int pos = j * RT_W;
    uint32_t d = (pos < 256 ? digit_w(k, pos, (256 - pos) < RT_W ? (256 - pos) : RT_W) : 0u) + carry;
    carry = d > 16 ? 1u : 0u;
    const bool neg = d > 16;
    if (neg) d = 32 - d;
    if (d) {
      P256Aff q;
      p256_ld_aff(q, tab + ((size_t)j * RT_ROW + (d - 1)) * P256_AFF_WORDS);
      if (neg) P256p::neg(q.y, q.y);
      p256_madd(acc, acc, q);
    }
  }
}
// Split commitments for the 34 jobs of a 0-bit repetition.  Several of them commit to the SAME value
// with different blinders (proveMult: A_z and A_4_1 both commit k_z, mult.ts:112-113; proveEquality:
// A_1 and A_2 both commit k, equality.ts:67-68), and C4 of a MultProof commits x y, which is the value of another job:
// i8 i9 = i10, i10 i10 = i11 and i10 i12 = i13 are computed as exactly these products (ItemScalarsTask), so C4 of
// MultProofs 1..3 shares the g-part of C10, C11, C13; C4 of MultProof 0 commits i7 i8, which is 1, or 0 when x1 = x2
// (invMod(0) = 0), and starts at its own value's table entry.  The g-parts v*g are computed once per distinct value
// (24 per item) and every job continues from its g-part with the 11 lookups of r*h.
#if defined(ZKA_PG_WAR256)
enum : int { GJOBS_PER_ITEM = 24, TOM_EXT_WORDS = 24 };
#else
enum : int { GJOBS_PER_ITEM = 24, TOM_EXT_WORDS = 36 };
#endif
// job index (0..33) -> index of its g-part (0..23), or -1: C4 of MultProof 0, whose value is 0 or 1
ZK_HD int item_gpart_of_job(int j) {
  if (j < 6) return j;                       // T1x T1y C8 C10 C11 C13
  if (j < 30) {                              // MultProof m: C4 Ax Ay Az A4_1 A4_2 -> (C10 C11 C13 of m - 1) 0 1 2 2 3
    const int m = (j - 6) / 6, u = (j - 6) % 6;
    if (u == 0) return m ? 2 + m : -1;
    return 6 + 4 * m + (u < 4 ? u - 1 : u - 2);
  }
  return 22 + ((j - 30) >> 1);               // EqualityProof e: A1, A2 share k
}
// g-part index (0..23) -> a job that carries its value scalar
ZK_HD int item_job_of_gpart(int g) {
  if (g < 6) return g;
  if (g < 22) {
    const int m = (g - 6) / 4, u = (g - 6) % 4;
    return 6 + 6 * m + (u < 3 ? u + 1 : 5);
  }
  return 30 + 2 * (g - 22);
}
// Which g-part each job of a batch continues from, for the item jobs (gk_n = 0: items of JOBS_PER_ITEM jobs and
// GJOBS_PER_ITEM g-parts) or for the Groth-Kohlweiss commitments (gk.ts:129-133, 173-176: rows of 4 gk_n slots cl, ca,
// cb, cd of the row's depth n_r, zero jobs behind them, and 2 gk_n g-parts, those of ca_i at i and of cd_i at gk_n + i).
// cl_i commits l_i in {0, 1} and cb_i commits l_i a_i, which is 0 or the value of ca_i, so only ca_i and cd_i are
// walked over g.  A job whose value is 0 or 1 starts at that value's window-0 entry (the identity or g) whichever
// g-part is named, and a job with no g-part (-1) always has such a value.
struct GpartLayout {
  int gk_n;                     // 0: item jobs; > 0: GK rows, the largest depth of the batch
  const uint32_t* ring_of;      // GK rows of a ring set: the ring of each row and the depth of each ring (else null)
  const uint32_t* ring_depth;
  ZK_HD int jobs() const { return gk_n ? 4 * gk_n : JOBS_PER_ITEM; }      // per item or row
  ZK_HD int gparts() const { return gk_n ? 2 * gk_n : GJOBS_PER_ITEM; }
  ZK_HD int depth(int row) const { return ring_of ? (int)ring_depth[ring_of[row]] : gk_n; }
  // the job whose value g-part g of `row` walks, or -1 (a row shallower than gk_n has no such g-part)
  ZK_HD int job_of_gpart(int row, int g) const {
    if (!gk_n) return item_job_of_gpart(g);
    const int n = depth(row), i = g % gk_n;
    return i < n ? (g < gk_n ? n : 3 * n) + i : -1;
  }
  // the g-part job j of `row` continues from, or -1
  ZK_HD int gpart_of_job(int row, int j) const {
    if (!gk_n) return item_gpart_of_job(j);
    const int n = depth(row);
    if (j < n || j >= 4 * n) return -1;     // cl_i, and the zero jobs
    const int i = j % n;
    return j < 3 * n ? i : gk_n + i;          // ca_i and cb_i: ca_i's g-part; cd_i: its own
  }
};
ZK_HD bool scalar_le_one(const uint32_t* v) { return (v[0] >> 1 | v[1] | v[2] | v[3] | v[4] | v[5] | v[6] | v[7]) == 0; }
#if defined(ZKA_PG_WAR256)
#include "zk_ops_war.cuh"
#else
// ===================================================================== tomEdwards256 tables
struct TomPowsTask {
  const uint32_t* base_aff;  // [nbase][18] image-curve affine (x', y), Montgomery
  uint32_t* pows;            // [nbase][nwin][36] extended (X,Y,T,Z): 2^bitpos(j) * base
  int nbase;
  FbShape sh;
  ZK_HD void operator()(int t) const {
    uint32_t x[9], y[9];
    ld<9>(x, base_aff + (size_t)t * TOM_AFF_WORDS);
    ld<9>(y, base_aff + (size_t)t * TOM_AFF_WORDS + 9);
    TomPt p;
    tom_from_affine(p, x, y);
    for (int j = 0; j < sh.nwin; j++) {
      uint32_t* o = pows + ((size_t)t * sh.nwin + j) * 36;
      st<9>(o, p.x); st<9>(o + 9, p.y); st<9>(o + 18, p.t); st<9>(o + 27, p.z);
      for (int k = 0; k < sh.width(j); k++) tom_dbl(p, p);
    }
  }
};
// The rows of ONE window are staged at a time (112 bytes per entry), so the staging buffer is bounded by the widest
// window and not by the table.
// rows of a window of w bits: proj store [d][27] = d * pow, d = 0 .. 2^(w-1)  (d = 0 is the identity)
struct TomRowsTask {
  const uint32_t* pow;    // [36]
  uint32_t* rows;
  int w;
  ZK_HD void operator()(int) const {
    TomPt p, acc;
    ld<9>(p.x, pow); ld<9>(p.y, pow + 9); ld<9>(p.t, pow + 18); ld<9>(p.z, pow + 27);
    tom_set_identity(acc);
    const int ne = fb_entries(w);
    for (int d = 0; d < ne; d++) {
      uint32_t* o = rows + (size_t)d * TOM_PROJ_WORDS;
      tom_st_xyz(o, acc.x, acc.y, acc.z);
      tom_add(acc, acc, p);
    }
  }
};
// Two-level construction of the same rows for wide windows (w > 9): first the 2^(w-9) + 1 "high" multiples
// m * 2^8 * P_j of every window (one thread per window), then, window by window, one thread per m walks the 256
// entries above it (the last m = 2^(w-9) is the top entry 2^(w-1) * P_j alone).  2^(w-9) + 256 sequential additions
// instead of 2^(w-1).
ZK_HD size_t tom_hi_offset(const FbShape& sh, int j) { return ((sh.offset(j) - (size_t)j) >> 8) + (size_t)j; }   // sum of 2^(w_i - 9) + 1 over i < j
struct TomRowsHiTask {
  const uint32_t* pows;   // [nwin][36]
  uint32_t* hi;           // window j at tom_hi_offset(j): [2^(w_j-9) + 1][36]
  FbShape sh;
  ZK_HD void operator()(int t) const {
    TomPt p, acc;
    const uint32_t* s = pows + (size_t)t * 36;
    ld<9>(p.x, s); ld<9>(p.y, s + 9); ld<9>(p.t, s + 18); ld<9>(p.z, s + 27);
    for (int k = 0; k < 8; k++) tom_dbl(p, p);
    tom_set_identity(acc);
    const int nh = 1 << (sh.width(t) - 9);
    for (int m = 0; m <= nh; m++) {
      uint32_t* o = hi + (tom_hi_offset(sh, t) + m) * 36;
      st<9>(o, acc.x); st<9>(o + 9, acc.y); st<9>(o + 18, acc.t); st<9>(o + 27, acc.z);
      tom_add(acc, acc, p);
    }
  }
};
struct TomRowsLoTask {
  const uint32_t* pow;    // [36]: the window's 2^bitpos * base
  const uint32_t* hi;     // [nh + 1][36]: the window's high multiples
  uint32_t* rows;         // [256 nh + 1][27]
  int nh;
  ZK_HD void operator()(int m) const {
    TomPt p, acc;
    ld<9>(p.x, pow); ld<9>(p.y, pow + 9); ld<9>(p.t, pow + 18); ld<9>(p.z, pow + 27);
    const uint32_t* h = hi + (size_t)m * 36;
    ld<9>(acc.x, h); ld<9>(acc.y, h + 9); ld<9>(acc.t, h + 18); ld<9>(acc.z, h + 27);
    uint32_t* out = rows + ((size_t)m << 8) * TOM_PROJ_WORDS;
    const int n = m < nh ? 256 : 1;
    for (int d = 0; d < n; d++) {
      uint32_t* o = out + (size_t)d * TOM_PROJ_WORDS;
      tom_st_xyz(o, acc.x, acc.y, acc.z);
      tom_add(acc, acc, p);
    }
  }
};
// Rows of a fixed-base table (E1 projective X:Y:Z) -> entries of the prover's a = -1 image curve
// E2 (zk_curves.cuh): (w, v) = (sqrt(-d1) X/Z, Z/Y), stored as (v - w, v + w, 2 d2 w v), canonical,
// one 128-byte line each.  Montgomery's trick over chunks of 16 entries on the products Y*Z.
struct TomTabE2Task {
  const uint32_t* proj;  // [count][27]
  uint32_t* pre;         // [count][32]
  int count;
  ZK_HD void operator()(int t) const {
    using F = Tomp;
    constexpr int CH = 16;
    const int lo = t * CH;
    int n = count - lo;
    if (n > CH) n = CH;
    if (n <= 0) return;
    uint32_t pf[CH][9];
    uint32_t acc[9], y[9], z[9], den[9];
    F::set_one(acc);
    for (int k = 0; k < n; k++) {
      const uint32_t* src = proj + (size_t)(lo + k) * TOM_PROJ_WORDS;
      uint32_t xx[9];
      tom_ld_xyz(xx, y, z, src);
      F::mul(den, y, z);
      F::mul(acc, acc, den);
      copy_n<9>(pf[k], acc);
    }
    uint32_t inv[9], s2[9], dd2[9];
    F::inv(inv, acc);
    tom_const(s2, TOM_SQRTND1);
    tom_const(dd2, TOM_2D2);
    for (int k = n - 1; k >= 0; k--) {
      const uint32_t* src = proj + (size_t)(lo + k) * TOM_PROJ_WORDS;
      uint32_t x[9], di[9], w[9], v[9], kk[9], ym[9], yp[9];
      tom_ld_xyz(x, y, z, src);
      F::mul(den, y, z);
      if (k > 0) F::mul(di, inv, pf[k - 1]); else copy_n<9>(di, inv);   // 1 / (Y Z)
      F::mul(inv, inv, den);
      F::mul(w, x, y);      // X Y
      F::mul(w, w, di);     // X / Z
      F::mul(w, w, s2);     // w
      F::sqr(v, z);
      F::mul(v, v, di);     // Z / Y
      F::mul(kk, w, v);
      F::mul(kk, kk, dd2);
      F::sub(ym, v, w);
      F::add(yp, v, w);
      F::reduce(ym); F::reduce(yp); F::reduce(kk);
      uint32_t* o = pre + (size_t)(lo + k) * TOM_PRE_WORDS;
      st<9>(o, ym); st<9>(o + 9, yp); st<9>(o + 18, kk);
      for (int i = 27; i < 32; i++) o[i] = 0;
    }
  }
};

// Batched normalisation of tomEdwards256 points -> E1 affine (x', y) Montgomery (+ optional 67-byte
// reference encoding of (x = x'/sqrt(a), y)).  e2 == 0: input is E1 projective (X:Y:Z);
// e2 == 1: input is (E, F, G, H) of the last addition of a commitment walk (tom2_madd_end):
// x' = E / (G sqrt(-d1)) = E H / (G H sqrt(-d1)), y = F / H = F G / (G H).
struct TomNormTask {
  const uint32_t* proj;  // [count][stride]: (X, Y, Z) or (E, F, G, H)
  uint32_t* aff;         // [count][18] or null
  uint8_t* bytes;        // [count][BSTRIDE] or null
  int count;
  int chunk;             // points per thread (<= NORM_CHUNK_MAX)
  int e2;
  int aff_mod, aff_lim;  // the E1 affine pair is produced only for points with (index % aff_mod) < aff_lim
  int stride;            // words per input slot: TOM_E2_WORDS or TOM_PROJ_WORDS (an (X, Y, Z) slot may be wider)
  ZK_HD static void canon2p(uint32_t* r) {   // value < 4p -> [0, p)
    uint32_t t[9], p2[9];
#pragma unroll
    for (int i = 0; i < 9; i++) p2[i] = (FpTom::p(i) << 1) | (i > 0 ? (FpTom::p(i - 1) >> 31) : 0u);
    uint32_t br = sub_n<9>(t, r, p2);
    csel_n<9>(r, br == 0, t, r);
    br = sub_p<FpTom>(t, r);
    csel_n<9>(r, br == 0, t, r);
  }
  ZK_HD void operator()(int t) const {
    using F = Tomp;
    const int lo = t * chunk;
    int n = count - lo;
    if (n > chunk) n = chunk;
    if (n <= 0) return;
    uint32_t pre[NORM_CHUNK_MAX][9];
    uint32_t acc[9], z[9], h[9], den[9];
    F::set_one(acc);
    for (int k = 0; k < n; k++) {
      const uint32_t* src = proj + (size_t)(lo + k) * stride;
      uint32_t xx[9], yy[9];
      if (e2) {
        tom_ld_efgh(xx, yy, z, h, src);
        F::mul(den, z, h);       // G H
      } else {
        tom_ld_xyz(xx, yy, den, src);
      }
      F::mul(acc, acc, den);   // Z != 0 (complete curve); G, H != 0 inside the prime-order subgroup
      copy_n<9>(pre[k], acc);
    }
    uint32_t inv[9], cxk[9], is2[9], one_plain[9];
    F::inv(inv, acc);
    tom_const(cxk, e2 ? TOM_INVSQRTND : TOM_INVSQRTA);   // 1 / sqrt(-d) or 1 / sqrt(a): x of the encoding
    tom_const(is2, TOM_INVSQRTND1);
    zero_n<9>(one_plain);
    one_plain[0] = 1;
    for (int k = n - 1; k >= 0; k--) {
      const uint32_t* src = proj + (size_t)(lo + k) * stride;
      uint32_t X[9], Y[9], di[9];
      if (e2) {                         // over den = G H:  x' sqrt(-d1) = E H / den,  y = F G / den
        tom_ld_efgh(X, Y, z, h, src);
        F::mul(den, z, h);
        F::mul(X, X, h);
        F::mul(Y, Y, z);
      } else {
        tom_ld_xyz(X, Y, den, src);
      }
      if (k > 0) F::mul(di, inv, pre[k - 1]); else copy_n<9>(di, inv);   // Montgomery residue of 1/den
      F::mul(inv, inv, den);
      if (bytes) {
        // D = 1/den as a PLAIN integer: a Montgomery product with it leaves Montgomery form, so the
        // reference coordinates come out without separate from_mont multiplications
        // e2: x = E H D / sqrt(-d),  y = F G D;  E1: x = X D / sqrt(a),  y = Y D
        uint32_t Dp[9], cx[9], cy[9];
        F::mul(Dp, di, one_plain);
        F::mul(cx, X, cxk);
        F::mul(cx, cx, Dp);
        F::mul(cy, Y, Dp);
        canon2p(cx);
        canon2p(cy);
        store_point_words<9, 33>(bytes + (size_t)(lo + k) * BSTRIDE, 0x04u, cx, cy);
      }
      if (aff && ((lo + k) % aff_mod) < aff_lim) {
        uint32_t x[9], y[9];
        F::mul(x, X, di);
        if (e2) F::mul(x, x, is2);     // x' = E / (G sqrt(-d1))
        F::mul(y, Y, di);
        uint32_t* a = aff + (size_t)(lo + k) * TOM_AFF_WORDS;
        st<9>(a, x);
        st<9>(a + 9, y);
      }
    }
  }
};

// entry |d| of window j of a signed-digit E2 table of shape sh ([total][32]), negated for a negative digit
ZK_HD void tom2_ld_entry(TomPre& q, const uint32_t* tab, const FbShape& sh, int j, uint32_t d, bool neg) {
  tom_ld_pre(q, tab + (sh.offset(j) + d) * TOM_PRE_WORDS);
  tom2_pre_neg(q, neg);
}

// Pedersen commitment in the proof group:  C = v*g + r*h   (pedersen.ts:53-58, gk.ts:88-92),
// both bases fixed => two positional tables, 2*nwin mixed additions, no doublings.  The walk starts at the entry of
// v's first window (tom2_from_pre, 1M) and, for the normaliser, ends with tom2_madd_end (3M): 1 + (2 nwin - 2) * 7 + 3
// products instead of 2 nwin * 7.  A zero digit selects entry 0, the identity.
struct TomCommitTask {
  const uint32_t* jv;    // [count][8] canonical value scalars (mod tom.order)
  const uint32_t* jr;    // [count][8] canonical blinders
  const uint32_t* gtab;  // [sh.total()][32]
  const uint32_t* htab;
  uint32_t* proj;        // [count][TOM_E2_WORDS] (E, F, G, H) -> TomNormTask{e2 = 1}; xyz: [count][TOM_PROJ_WORDS]
  FbShape sh;
  int xyz = 0;           // 1: a full last addition, E2 (W : V : Z) for readers other than the normaliser (pg_fixed_to_msm)
  ZK_HD void operator()(int t) const {
    uint32_t v[8], r[8];
    ld<8>(v, jv + (size_t)t * 8);
    ld<8>(r, jr + (size_t)t * 8);
    uint32_t cv = 0, cr = 0;
    bool nv, nr;
    TomPre q;
    uint32_t dv = signed_digit(v, 0, sh, cv, nv);
    tom2_ld_entry(q, gtab, sh, 0, dv, nv);
    TomPt acc;
    tom2_from_pre(acc, q);
    for (int j = 0;; j++) {
      const uint32_t dr = signed_digit(r, j, sh, cr, nr);
      tom2_ld_entry(q, htab, sh, j, dr, nr);
      if (j == sh.nwin - 1) break;
      tom2_madd<true>(acc, acc, q);     // a = -1 image curve E2: 7M per lookup
      dv = signed_digit(v, j + 1, sh, cv, nv);
      tom2_ld_entry(q, gtab, sh, j + 1, dv, nv);
      tom2_madd<true>(acc, acc, q);
    }
    if (xyz) {
      tom2_madd<false>(acc, acc, q);
      tom_st_xyz(proj + (size_t)t * TOM_PROJ_WORDS, acc.x, acc.y, acc.z);
    } else {
      TomEfgh e;
      tom2_madd_end(e, acc, q);
      tom_st_efgh(proj + (size_t)t * TOM_E2_WORDS, e);
    }
  }
};

struct TomCommitGTask {   // one thread per g-part of GpartLayout: K = v*g as an extended E2 point, from v's first entry
  const uint32_t* jv;     // [rows * lay.jobs()][8]
  const uint32_t* gtab;
  uint32_t* ext;          // [rows * lay.gparts()][36]
  FbShape sh;
  GpartLayout lay;
  ZK_HD void operator()(int t) const {
    const int row = t / lay.gparts(), jb = lay.job_of_gpart(row, t % lay.gparts());
    if (jb < 0) return;
    uint32_t v[8];
    ld<8>(v, jv + ((size_t)row * lay.jobs() + jb) * 8);
    uint32_t carry = 0;
    bool neg;
    TomPre q;
    const uint32_t d0 = signed_digit(v, 0, sh, carry, neg);
    tom2_ld_entry(q, gtab, sh, 0, d0, neg);
    TomPt acc;
    tom2_from_pre<TompCommit>(acc, q);
#pragma unroll 1
    for (int j = 1; j < sh.nwin; j++) {
      const uint32_t d = signed_digit(v, j, sh, carry, neg);
      tom2_ld_entry(q, gtab, sh, j, d, neg);
      tom2_madd<true, TompCommit>(acc, acc, q);
    }
    uint32_t* o = ext + (size_t)t * TOM_EXT_WORDS;
    st<9>(o, acc.x); st<9>(o + 9, acc.y); st<9>(o + 18, acc.t); st<9>(o + 27, acc.z);
  }
};
struct TomCommitHTask {   // one thread per job: C = K + r*h, ending in tom2_madd_end for the normaliser
  const uint32_t* jv;     // [rows * lay.jobs()][8]
  const uint32_t* jr;
  const uint32_t* gtab;
  const uint32_t* htab;
  const uint32_t* ext;    // [rows * lay.gparts()][36]
  uint32_t* proj;         // [rows * lay.jobs()][TOM_E2_WORDS]  (E, F, G, H) -> TomNormTask{e2 = 1}
  FbShape sh;
  GpartLayout lay;
  ZK_HD void operator()(int t) const {
    const int row = t / lay.jobs(), g = lay.gpart_of_job(row, t % lay.jobs());
    uint32_t v[8], r[8];
    ld<8>(v, jv + (size_t)t * 8);
    TomPt acc;
    TomPre q;
    if (g < 0 || scalar_le_one(v)) {   // K = v*g is the entry of v in window 0 (entry 0 is the identity)
      tom2_ld_entry(q, gtab, sh, 0, v[0], false);
      tom2_from_pre<TompCommit>(acc, q);
    } else {
      const uint32_t* s = ext + ((size_t)row * lay.gparts() + g) * TOM_EXT_WORDS;
      ld<9>(acc.x, s); ld<9>(acc.y, s + 9); ld<9>(acc.t, s + 18); ld<9>(acc.z, s + 27);
    }
    ld<8>(r, jr + (size_t)t * 8);
    uint32_t carry = 0;
    bool neg;
#pragma unroll 1
    for (int j = 0; j < sh.nwin - 1; j++) {
      const uint32_t d = signed_digit(r, j, sh, carry, neg);
      tom2_ld_entry(q, htab, sh, j, d, neg);
      tom2_madd<true, TompCommit>(acc, acc, q);
    }
    const uint32_t d = signed_digit(r, sh.nwin - 1, sh, carry, neg);
    tom2_ld_entry(q, htab, sh, sh.nwin - 1, d, neg);
    TomEfgh e;
    tom2_madd_end<TompCommit>(e, acc, q);
    tom_st_efgh(proj + (size_t)t * TOM_E2_WORDS, e);
  }
};

#if !defined(ZKA_HOSTSIM) && defined(ZKA_COMMIT_MINBLOCKS)
template <> struct TaskMinBlocks<TomCommitHTask> { static constexpr int value = ZKA_COMMIT_MINBLOCKS; };
template <> struct TaskMinBlocks<TomCommitGTask> { static constexpr int value = ZKA_COMMIT_MINBLOCKS; };
template <> struct TaskMinBlocks<TomCommitTask> { static constexpr int value = ZKA_COMMIT_MINBLOCKS; };
#endif

#endif   // ZKA_PG_WAR256

// ============================================================================ Groth-Kohlweiss sums
// sum over the 2^k ring entries i of block `blk` of coef_i * prod_j (bit_j(i) ? fo[j] : fz[j]),
// coef_i = vw ? (vw - v_i) : v_i  (gk.ts:141-171 prover, gk.ts:239-250 verifier).  The product is walked
// incrementally over the binary counter of the low k bits (about 3 multiplications per entry); the high
// n-k bits are fixed by the block index.  k = n, blk = 0 is the whole ring in one call; large rings are
// cut into blocks of 2^GK_BLOCK_BITS entries, one thread each, and summed afterwards.
enum : int { GK_BLOCK_BITS = 10 };
ZK_HD int gk_block_bits(int n) { return n < GK_BLOCK_BITS ? n : GK_BLOCK_BITS; }
ZK_HD void gk_block_sum(uint32_t* acc, const uint32_t* ring_m, const uint32_t (*fz)[8], const uint32_t (*fo)[8], int n,
                        int k, uint32_t blk, const uint32_t* vw) {
  using F = Tomq;
  uint32_t P[21][8];
  F::set_one(P[n]);
  for (int j = n - 1; j >= k; j--) F::mul(P[j], P[j + 1], ((blk >> (j - k)) & 1u) ? fo[j] : fz[j]);
  for (int j = k - 1; j >= 0; j--) F::mul(P[j], P[j + 1], fz[j]);
  zero_n<8>(acc);
  const size_t base = (size_t)blk << k;
  const uint32_t cnt = 1u << k;
  for (uint32_t l = 0;;) {
    uint32_t vi[8], term[8];
    ld<8>(vi, ring_m + (base + l) * 8);
    if (vw) F::sub(vi, vw, vi);
    F::mul(term, vi, P[0]);
    F::add(acc, acc, term);
    l++;
    if (l == cnt) break;
    // lowest set bit of the new l: bits below it are 0, it is 1, bits above unchanged
    int tz = 0;
    while (!((l >> tz) & 1u)) tz++;
    F::mul(P[tz], P[tz + 1], fo[tz]);
    for (int j = tz - 1; j >= 0; j--) F::mul(P[j], P[j + 1], fz[j]);
  }
}

// ================================================================================== hashing
// Streams `npts` encoded points (given as (pointer, length) by a functor) through SHA-256.
// Encodings are fetched one point ahead: five 16-byte loads from a 16-byte aligned address (every staging slot; the
// last block also holds the encoding's final bytes, so the load stays inside memory the encoding occupies), 17
// word loads from another 4-byte aligned one (proof rows), bytes otherwise.
ZK_HD bool hash_pt_fetch(uint32_t* t, const uint8_t* p, int len) {
  if (((size_t)p & 3) || len < 64 || len > 68) return false;
  if (aligned16(p)) {
#pragma unroll
    for (int j = 0; j < 4; j++) ld4(t + 4 * j, p + 16 * j);
    t[16] = len > 64 ? *reinterpret_cast<const uint32_t*>(p + 64) : 0u;
    return true;
  }
  const uint32_t* q = reinterpret_cast<const uint32_t*>(p);
#pragma unroll
  for (int j = 0; j < 17; j++) t[j] = (4 * j < len) ? q[j] : 0u;
  return true;
}
template <class Src>
ZK_HD void hash_points80(uint32_t* c3, const Src& src, int npts) {
  Sha256 h;
  h.init();
  uint32_t nx[17], cu[17];
  int nlen = 0;
  const uint8_t* np = npts > 0 ? src(0, nlen) : nullptr;
  bool nfast = npts > 0 && hash_pt_fetch(nx, np, nlen);
  for (int i = 0; i < npts; i++) {
    const uint8_t* p = np;
    const int len = nlen;
    const bool fast = nfast;
#pragma unroll
    for (int j = 0; j < 17; j++) cu[j] = nx[j];
    if (i + 1 < npts) {
      np = src(i + 1, nlen);
      nfast = hash_pt_fetch(nx, np, nlen);
    }
    if (fast) h.feed17(cu, len);
    else h.update(p, len);
  }
  h.final80(c3);
}

// challenge (80 bit, c3) as a canonical 8-limb scalar
ZK_HD void challenge_to_limbs(uint32_t* r, const uint32_t* c3) {
  zero_n<8>(r);
  r[0] = c3[0]; r[1] = c3[1]; r[2] = c3[2];
}

// the encoded point (N = 65 or 67 bytes) at src as little-endian stream words w[0, 20): five 16-byte loads from a
// 16-byte aligned address (every BSTRIDE slot), word loads from another 4-byte aligned one, bytes otherwise
template <int N>
ZK_HD void load_point(uint32_t* w, const uint8_t* src) {
  if (aligned16(src)) {
#pragma unroll
    for (int j = 0; j < BSTRIDE / 16; j++) ld4(w + 4 * j, src + 16 * j);
  } else if (((size_t)src & 3) == 0) {
    const uint32_t* sw = reinterpret_cast<const uint32_t*>(src);
#pragma unroll
    for (int j = 0; j < BSTRIDE / 4; j++) w[j] = 4 * j < N ? sw[j] : 0u;
  } else {
#pragma unroll
    for (int j = 0; j < BSTRIDE / 4; j++) {
      uint32_t v = 0;
#pragma unroll
      for (int t = 0; t < 4; t++)
        if (4 * j + t < N) v |= (uint32_t)src[4 * j + t] << (8 * t);
      w[j] = v;
    }
  }
}

// Writes one contiguous output region of any alignment as a byte stream.  Pieces (encoded points, scalars, single
// bytes) are appended in order as little-endian stream words; every whole 16-byte block of the region is one 16-byte
// store, assembled in registers with a run-time byte shift.  The region's first and last blocks may be shared with
// neighbouring regions written by other threads (MultProof m and m + 1, a repetition head and its body): only the
// region's own bytes of them are stored, with 4- and 1-byte stores.  All register indices are static.
struct ByteWriter {
  uint8_t* blk;   // the 16-byte block being assembled
  uint32_t q[4];  // its bytes below `fill`, little-endian; zero above
  int fill;       // bytes of the block decided so far
  int lead;       // bytes [0, lead) of the block belong to whatever precedes the region (first block only)
  ZK_HD explicit ByteWriter(uint8_t* dst) : blk(dst - ((size_t)dst & 15)), fill((int)((size_t)dst & 15)), lead(fill) {
    q[0] = q[1] = q[2] = q[3] = 0;
  }
  ZK_HD static uint32_t funnel(uint32_t lo, uint32_t hi, int sh) {   // high word of (hi:lo) << sh, sh in [0, 32)
#if defined(__CUDA_ARCH__)
    return __funnelshift_l(lo, hi, sh);
#else
    return (uint32_t)((((uint64_t)hi << 32) | lo) >> (32 - sh));
#endif
  }
  ZK_HD void store_part(int lo, int hi) const {   // bytes [lo, hi) of the current block
#pragma unroll
    for (int w = 0; w < 4; w++) {
      if (lo <= 4 * w && 4 * w + 4 <= hi) {
        *reinterpret_cast<uint32_t*>(blk + 4 * w) = q[w];
      } else {
#pragma unroll
        for (int t = 0; t < 4; t++)
          if (lo <= 4 * w + t && 4 * w + t < hi) blk[4 * w + t] = (uint8_t)(q[w] >> (8 * t));
      }
    }
  }
  // append nb (1..16) bytes held in c[0, 4)
  ZK_HD void chunk(const uint32_t* c, int nb) {
    uint32_t m[4];
#pragma unroll
    for (int i = 0; i < 4; i++) {
      const int k = nb - 4 * i;   // bytes of word i that belong to the chunk
      m[i] = k >= 4 ? c[i] : k <= 0 ? 0u : c[i] & ((1u << (8 * k)) - 1u);
    }
    const int sh = 8 * (fill & 3), ws = fill >> 2;
    uint32_t d[5];
    d[0] = sh ? m[0] << sh : m[0];
#pragma unroll
    for (int i = 1; i < 4; i++) d[i] = funnel(m[i - 1], m[i], sh);
    d[4] = sh ? m[3] >> (32 - sh) : 0u;
    uint32_t e[8];
#pragma unroll
    for (int k = 0; k < 8; k++) {
      uint32_t v = 0;
#pragma unroll
      for (int s = 0; s < 4; s++)
        if (k - s >= 0 && k - s <= 4) v = ws == s ? d[k - s] : v;
      e[k] = v;
    }
#pragma unroll
    for (int k = 0; k < 4; k++) q[k] |= e[k];
    fill += nb;
    if (fill >= 16) {
      if (lead == 0) st4(blk, q); else store_part(lead, 16);
      blk += 16;
      lead = 0;
      fill -= 16;
#pragma unroll
      for (int k = 0; k < 4; k++) q[k] = e[4 + k];
    }
  }
  // append the first NB bytes of the stream words w[0, ceil(NB / 4))
  template <int NB>
  ZK_HD void put(const uint32_t* w) {
#pragma unroll
    for (int c = 0; c < (NB + 15) / 16; c++) {
      uint32_t v[4];
#pragma unroll
      for (int i = 0; i < 4; i++) v[i] = 16 * c + 4 * i < NB ? w[4 * c + i] : 0u;
      chunk(v, NB - 16 * c < 16 ? NB - 16 * c : 16);
    }
  }
  ZK_HD void put_byte(uint32_t b) {
    const uint32_t v[4] = {b, 0u, 0u, 0u};
    chunk(v, 1);
  }
  // an encoded point of N bytes (65 or 67) from a BSTRIDE slot
  template <int N>
  ZK_HD void put_point(const uint8_t* src) {
    uint32_t w[BSTRIDE / 4];
    load_point<N>(w, src);
    put<N>(w);
  }
  // a canonical 8-limb scalar as a big-endian field of LEN bytes (32 or 33)
  template <int LEN>
  ZK_HD void put_scalar(const uint32_t* c) {
    uint32_t w[9];
#pragma unroll
    for (int j = 0; j < 9; j++) {
      uint32_t v = 0;
#pragma unroll
      for (int t = 0; t < 4; t++) {
        const int k = 4 * j + t;               // stream position
        const int pos = LEN - 1 - k;           // byte significance
        if (k < LEN && pos >= 0 && pos < 32) v |= ((c[pos >> 2] >> (8 * (pos & 3))) & 0xffu) << (8 * t);
      }
      w[j] = v;
    }
    put<LEN>(w);
  }
  // store the bytes of the last, partly filled block; the writer is done
  ZK_HD void finish() {
    if (fill > lead) store_part(lead, fill);
  }
};

}  // namespace zk
