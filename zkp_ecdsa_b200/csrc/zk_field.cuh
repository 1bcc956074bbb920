// zk_field.cuh — Montgomery arithmetic for the four moduli of the ZKAttest hot path.
//
// Replaces the reference's BigInt `(a*b) % p`, posMod, invMod, expMod
// (/root/reference/src/bignum/big.ts:36-119) with fixed-width 32-bit-limb Montgomery
// arithmetic that lives in registers:
//   FpP256  p256.p  (8 limbs, strict  [0,p))   P-256 coordinates AND tomEdwards256 scalars
//                                              (tom.order == p256.p, src/curves/instances.ts:48)
//   FnP256  p256.n  (8 limbs, strict  [0,n))   P-256 scalars
//   FpTom   tom.p   (9 limbs, LAZY    [0,2^13 p)) tomEdwards256 coordinates; 258-bit prime,
//                                              R = 2^288 leaves 30 bits of headroom so
//                                              add/sub never reduce and mul needs no final
//                                              conditional subtraction.
// All code is __host__ __device__ so the identical arithmetic can be exercised by the
// host-side simulator used in CPU tests (tests/hostsim); the product library is the
// nvcc/sm_90a build only.
#pragma once
#include <stdint.h>
#include "zk_field_consts.inc"

#if defined(__CUDACC__)
#define ZK_HD __host__ __device__ __forceinline__
#define ZK_HDN __host__ __device__ __noinline__
#else
#define ZK_HD inline __attribute__((always_inline))
#define ZK_HDN __attribute__((noinline))
#endif

namespace zk {

// ------------------------------------------------------------------------------------
// Field descriptors.  Limbs little-endian (limb 0 = least significant 32 bits).
// ------------------------------------------------------------------------------------
#define ZK_FIELD_DESC(NAME, PFX, NL, LAZY)                                   \
  struct NAME {                                                              \
    static constexpr int N = NL;                                             \
    static constexpr bool kLazy = LAZY;                                      \
    static constexpr uint32_t kN0Inv = PFX##_N0INV;                          \
    ZK_HD static constexpr uint32_t p(int i) {                               \
      constexpr uint32_t t[NL] = PFX##_P;                                    \
      return t[i];                                                           \
    }                                                                        \
    ZK_HD static constexpr uint32_t rr(int i) {                              \
      constexpr uint32_t t[NL] = PFX##_RR;                                   \
      return t[i];                                                           \
    }                                                                        \
    ZK_HD static constexpr uint32_t one(int i) {                             \
      constexpr uint32_t t[NL] = PFX##_ONE;                                  \
      return t[i];                                                           \
    }                                                                        \
  };
ZK_FIELD_DESC(FpP256, ZK_P256P, 8, false)
ZK_FIELD_DESC(FnP256, ZK_P256N, 8, false)
ZK_FIELD_DESC(FpTom, ZK_TOMP, 9, true)
ZK_FIELD_DESC(FpWar, ZK_WARP, 8, false)   // war256 coordinates (instances.ts:34-41), strict [0,p), generic CIOS
#undef ZK_FIELD_DESC

template <int N>
struct Fe {
  uint32_t v[N];
};
using Fe8 = Fe<8>;
using Fe9 = Fe<9>;

// ------------------------------------------------------------------------------------
// Multi-word helpers (portable 64-bit carries; nvcc lowers them to IADD3/IADD3.X)
// ------------------------------------------------------------------------------------
template <int N>
ZK_HD uint32_t add_n(uint32_t* r, const uint32_t* a, const uint32_t* b) {
  uint64_t c = 0;
#pragma unroll
  for (int i = 0; i < N; i++) {
    c += (uint64_t)a[i] + b[i];
    r[i] = (uint32_t)c;
    c >>= 32;
  }
  return (uint32_t)c;
}
template <int N>
ZK_HD uint32_t sub_n(uint32_t* r, const uint32_t* a, const uint32_t* b) {
  int64_t c = 0;
#pragma unroll
  for (int i = 0; i < N; i++) {
    c += (int64_t)a[i] - (int64_t)b[i];
    r[i] = (uint32_t)c;
    c >>= 32;  // arithmetic shift: 0 or -1
  }
  return (uint32_t)(c & 1);  // borrow
}
template <class F>
ZK_HD uint32_t sub_p(uint32_t* r, const uint32_t* a) {  // r = a - p, returns borrow
  int64_t c = 0;
#pragma unroll
  for (int i = 0; i < F::N; i++) {
    c += (int64_t)a[i] - (int64_t)F::p(i);
    r[i] = (uint32_t)c;
    c >>= 32;
  }
  return (uint32_t)(c & 1);
}
template <class F>
ZK_HD bool geq_p(const uint32_t* a) {
#pragma unroll
  for (int i = F::N - 1; i >= 0; i--) {
    if (a[i] > F::p(i)) return true;
    if (a[i] < F::p(i)) return false;
  }
  return true;
}
template <int N>
ZK_HD bool is_zero_n(const uint32_t* a) {
  uint32_t o = 0;
#pragma unroll
  for (int i = 0; i < N; i++) o |= a[i];
  return o == 0;
}
template <int N>
ZK_HD bool eq_n(const uint32_t* a, const uint32_t* b) {
  uint32_t o = 0;
#pragma unroll
  for (int i = 0; i < N; i++) o |= a[i] ^ b[i];
  return o == 0;
}
template <int N>
ZK_HD void copy_n(uint32_t* r, const uint32_t* a) {
#pragma unroll
  for (int i = 0; i < N; i++) r[i] = a[i];
}
template <int N>
ZK_HD void zero_n(uint32_t* r) {
#pragma unroll
  for (int i = 0; i < N; i++) r[i] = 0;
}
template <int N>
ZK_HD void csel_n(uint32_t* r, bool c, const uint32_t* a, const uint32_t* b) {  // r = c ? a : b
#pragma unroll
  for (int i = 0; i < N; i++) r[i] = c ? a[i] : b[i];
}

}  // namespace zk
#include "zk_field_ptx.cuh"   // sm_90a multiplier kernels (device only)
namespace zk {

#if defined(__CUDA_ARCH__) && !defined(ZKA_NO_PTX_MUL)
// non-inlined generic 8-limb Montgomery product (defined below Field): the war256 coordinate field has no special
// multiplier; inlining the generic CIOS at each of the 13 products of a point addition bloats the kernels the way the
// first inlined tomEdwards256 multiplier did (instruction-fetch stalls)
namespace ptx {
template <class F> static __device__ __noinline__ V8 cios8_mul_fn(V8 a, V8 b);
}
#endif
template <class A, class B> struct same_t { static constexpr bool value = false; };
template <class A> struct same_t<A, A> { static constexpr bool value = true; };

// ------------------------------------------------------------------------------------
// Field operations
// ------------------------------------------------------------------------------------
template <class F>
struct Field {
  static constexpr int N = F::N;

  // canonical reduce of a lazy value (< 2^14 p) or a strict value (< 2p) into [0,p)
  ZK_HD static void reduce(uint32_t* a) {
    if (F::kLazy) {
      // value < 2^14 p: subtract 2^k p for k = 13..0 when possible (branch-free selects)
#pragma unroll 1
      for (int k = 13; k >= 0; k--) {
        uint32_t pk[N];
#pragma unroll
        for (int i = 0; i < N; i++) {
          uint32_t lo = F::p(i) << k;
          uint32_t hi = (i > 0 && k > 0) ? (F::p(i - 1) >> (32 - k)) : 0u;
          pk[i] = lo | hi;
        }
        uint32_t t[N];
        uint32_t br = sub_n<N>(t, a, pk);
        csel_n<N>(a, br == 0, t, a);
      }
    } else {
      uint32_t t[N];
      uint32_t br = sub_p<F>(t, a);
      csel_n<N>(a, br == 0, t, a);
    }
  }

  ZK_HD static void add(uint32_t* r, const uint32_t* a, const uint32_t* b) {
    if (F::kLazy) {
      add_n<N>(r, a, b);
    } else {
      uint32_t s[N], t[N];
      uint32_t c = add_n<N>(s, a, b);
      uint32_t br = sub_p<F>(t, s);
      csel_n<N>(r, (c != 0) || (br == 0), t, s);
    }
  }
  // lazy: r = a + 8p - b  (requires b < 8p)
  ZK_HD static void sub(uint32_t* r, const uint32_t* a, const uint32_t* b) {
    if (F::kLazy) {
      uint32_t p8[N];
#pragma unroll
      for (int i = 0; i < N; i++) p8[i] = (F::p(i) << 3) | (i > 0 ? (F::p(i - 1) >> 29) : 0u);
      uint32_t t[N];
      add_n<N>(t, a, p8);
      sub_n<N>(r, t, b);
    } else {
      uint32_t s[N], t[N];
      uint32_t br = sub_n<N>(s, a, b);
      uint32_t pp[N];
#pragma unroll
      for (int i = 0; i < N; i++) pp[i] = F::p(i);
      add_n<N>(t, s, pp);
      csel_n<N>(r, br != 0, t, s);
    }
  }
  ZK_HD static void neg(uint32_t* r, const uint32_t* a) {
    uint32_t z[N];
    zero_n<N>(z);
    sub(r, z, a);
  }
  ZK_HD static void dbl(uint32_t* r, const uint32_t* a) { add(r, a, a); }

  // Montgomery product r = a*b/R mod p  (CIOS).  r may alias a or b.
  ZK_HD static void mul(uint32_t* r, const uint32_t* a, const uint32_t* b) {
#if defined(__CUDA_ARCH__) && !defined(ZKA_NO_PTX_MUL)
    // product-scanning PTX kernels for the two hot moduli (zk_field_ptx.cuh)
    if (same_t<F, FpTom>::value) { ptx::tom_mul(r, a, b); return; }
    if (same_t<F, FpP256>::value) { ptx::p256_mul(r, a, b); return; }
    if (same_t<F, FpWar>::value) {
      ptx::V8 x, y;
#pragma unroll
      for (int i = 0; i < 8; i++) { x.v[i] = a[i]; y.v[i] = b[i]; }
      const ptx::V8 z = ptx::cios8_mul_fn<FpWar>(x, y);
#pragma unroll
      for (int i = 0; i < 8; i++) r[i] = z.v[i];
      return;
    }
#endif
    mul_generic(r, a, b);
  }
  // generic CIOS (any modulus of N limbs)
  ZK_HD static void mul_generic(uint32_t* r, const uint32_t* a, const uint32_t* b) {
    uint32_t t[N + 2];
#pragma unroll
    for (int i = 0; i < N + 2; i++) t[i] = 0;
#pragma unroll
    for (int i = 0; i < N; i++) {
      uint64_t c = 0;
      const uint32_t bi = b[i];
#pragma unroll
      for (int j = 0; j < N; j++) {
        uint64_t s = (uint64_t)a[j] * bi + t[j] + c;
        t[j] = (uint32_t)s;
        c = s >> 32;
      }
      uint64_t s = (uint64_t)t[N] + c;
      t[N] = (uint32_t)s;
      t[N + 1] = (uint32_t)(s >> 32);
      const uint32_t m = t[0] * F::kN0Inv;
      c = ((uint64_t)m * F::p(0) + t[0]) >> 32;
#pragma unroll
      for (int j = 1; j < N; j++) {
        uint64_t s2 = (uint64_t)m * F::p(j) + t[j] + c;
        t[j - 1] = (uint32_t)s2;
        c = s2 >> 32;
      }
      s = (uint64_t)t[N] + c;
      t[N - 1] = (uint32_t)s;
      t[N] = t[N + 1] + (uint32_t)(s >> 32);
    }
    if (F::kLazy) {
      copy_n<N>(r, t);  // < a*b/R + p < 2p for inputs < 2^13 p
    } else {
      uint32_t u[N];
      uint32_t br = sub_p<F>(u, t);
      csel_n<N>(r, (t[N] != 0) || (br == 0), u, t);
    }
  }
  ZK_HD static void sqr(uint32_t* r, const uint32_t* a) {
#if defined(__CUDA_ARCH__) && !defined(ZKA_NO_PTX_MUL)
    if (same_t<F, FpP256>::value) { ptx::p256_sqr(r, a); return; }   // 36 products instead of 64
#endif
    mul(r, a, a);
  }

  ZK_HD static void set_one(uint32_t* r) {
#pragma unroll
    for (int i = 0; i < N; i++) r[i] = F::one(i);
  }
  ZK_HD static void to_mont(uint32_t* r, const uint32_t* a) {
    uint32_t rr[N];
#pragma unroll
    for (int i = 0; i < N; i++) rr[i] = F::rr(i);
    mul(r, a, rr);
  }
  // out of Montgomery form AND canonical
  ZK_HD static void from_mont(uint32_t* r, const uint32_t* a) {
    uint32_t o[N];
    zero_n<N>(o);
    o[0] = 1;
    mul(r, a, o);
    if (F::kLazy) {
      // a*1/R + p < 2p for any legal lazy input (a < 2^13 p << R): two conditional subtractions
      // (2p, p) are more than enough; the generic 14-step ladder of reduce() is not needed here
      uint32_t t[N], p2[N];
#pragma unroll
      for (int i = 0; i < N; i++) p2[i] = (F::p(i) << 1) | (i > 0 ? (F::p(i - 1) >> 31) : 0u);
      uint32_t br = sub_n<N>(t, r, p2);
      csel_n<N>(r, br == 0, t, r);
      br = sub_p<F>(t, r);
      csel_n<N>(r, br == 0, t, r);
    } else {
      reduce(r);
    }
  }
  // canonical zero test of a (possibly lazy) Montgomery value
  ZK_HD static bool is_zero(const uint32_t* a) {
    uint32_t t[N];
    copy_n<N>(t, a);
    reduce(t);
    return is_zero_n<N>(t);
  }
  ZK_HD static bool eq(const uint32_t* a, const uint32_t* b) {
    uint32_t t[N], u[N];
    copy_n<N>(t, a);
    copy_n<N>(u, b);
    reduce(t);
    reduce(u);
    return eq_n<N>(t, u);
  }

  // r = a^(p-2) (Fermat inverse), a in Montgomery form; returns 0 for a == 0.  Kept as the
  // cross-check of inv() in the field-op tests (zka_field_op_batch op 4).
  static ZK_HDN void inv_fermat(uint32_t* r, const uint32_t* a) {
    uint32_t e[N];
#pragma unroll
    for (int i = 0; i < N; i++) e[i] = F::p(i);
    e[0] -= 2;  // p is odd and p(0) >= 2 for all our moduli
    uint32_t acc[N], base[N];
    set_one(acc);
    copy_n<N>(base, a);
    int top = N * 32 - 1;
    while (top > 0 && !((e[top >> 5] >> (top & 31)) & 1)) top--;
#pragma unroll 1
    for (int bit = top; bit >= 0; bit--) {
      sqr(acc, acc);
      if ((e[bit >> 5] >> (bit & 31)) & 1) mul(acc, acc, base);
    }
    copy_n<N>(r, acc);
  }

  // Modular inverse of a Montgomery residue (0 -> 0, like the reference's invEuclid,
  // /root/reference/src/bignum/big.ts:112-119).  Kaliski's binary "almost inverse"
  // (u, v, r, s) iteration, written branch-free so a warp stays converged inside an iteration:
  // ~1.4 * bitlen(p) rounds of shifts / adds / selects on N+1 limbs — ALU-pipe work worth about a
  // quarter of the 380-multiplication Fermat ladder — followed by four Montgomery products that
  // turn  A^-1 2^k  (A = a = xR)  into  x^-1 R.
  static ZK_HDN void inv(uint32_t* out, const uint32_t* a) {
    constexpr int L = N + 1;
    uint32_t u[L], v[L], r[L], s[L];
    {
      uint32_t t[N];
      copy_n<N>(t, a);
      reduce(t);                       // canonical A in [0, p)
#pragma unroll
      for (int i = 0; i < N; i++) { u[i] = F::p(i); v[i] = t[i]; r[i] = 0; s[i] = 0; }
      u[N] = 0; v[N] = 0; r[N] = 0; s[N] = 0;
      s[0] = 1;
    }
    if (is_zero_n<L>(v)) { zero_n<N>(out); return; }
    int k = 0;
#pragma unroll 1
    while (!is_zero_n<L>(v)) {
      uint32_t dm[L], dn[L], sm[L];
      const uint32_t bor = sub_n<L>(dm, u, v);     // u - v
      sub_n<L>(dn, v, u);                          // v - u
      add_n<L>(sm, r, s);
      const bool ue = (u[0] & 1u) == 0, ve = (v[0] & 1u) == 0;
      const bool gt = (bor == 0) && !is_zero_n<L>(dm);
      const bool cA = ue, cB = !ue && ve, cC = !ue && !ve && gt, cD = !ue && !ve && !gt;
      const bool su = cA || cC;                    // the u side is halved, s doubled
      const bool sv = cB || cD;                    // the v side is halved, r doubled
      uint32_t nu[L], nv[L], nr[L], ns[L];
#pragma unroll
      for (int i = 0; i < L; i++) {
        const uint32_t uu = cC ? dm[i] : u[i], uh = cC ? (i + 1 < L ? dm[i + 1] : 0u) : (i + 1 < L ? u[i + 1] : 0u);
        const uint32_t vv = cD ? dn[i] : v[i], vh = cD ? (i + 1 < L ? dn[i + 1] : 0u) : (i + 1 < L ? v[i + 1] : 0u);
        nu[i] = su ? ((uu >> 1) | (uh << 31)) : u[i];
        nv[i] = sv ? ((vv >> 1) | (vh << 31)) : v[i];
        const uint32_t rl = i > 0 ? r[i - 1] : 0u, sl = i > 0 ? s[i - 1] : 0u;
        nr[i] = cC ? sm[i] : (sv ? ((r[i] << 1) | (rl >> 31)) : r[i]);
        ns[i] = cD ? sm[i] : (su ? ((s[i] << 1) | (sl >> 31)) : s[i]);
      }
#pragma unroll
      for (int i = 0; i < L; i++) { u[i] = nu[i]; v[i] = nv[i]; r[i] = nr[i]; s[i] = ns[i]; }
      k++;
    }
    // r < 2p:  r -= p if r >= p;  result rr = p - r = A^-1 2^k mod p
    uint32_t pp[L], t[L];
#pragma unroll
    for (int i = 0; i < N; i++) pp[i] = F::p(i);
    pp[N] = 0;
    uint32_t br = sub_n<L>(t, r, pp);
    csel_n<L>(r, br == 0, t, r);
    sub_n<L>(t, pp, r);
    uint32_t rr[N];
    copy_n<N>(rr, t);
    // x^-1 R = rr * 2^(2m - k), m = 32 N:  two (R^2, 2^e) pairs of Montgomery products
    int e = 2 * 32 * N - k;
    const int emax = (F::p(N - 1) >> 31) ? 32 * N - 1 : 32 * (N - 1);   // 2^emax < p for our moduli
    int e1 = e < emax ? e : emax, e2 = e - e1;
    uint32_t rr2[N], pw[N];
#pragma unroll
    for (int i = 0; i < N; i++) rr2[i] = F::rr(i);
    mul(rr, rr, rr2);
    zero_n<N>(pw);
    pw[e1 >> 5] = 1u << (e1 & 31);
    mul(rr, rr, pw);
    mul(rr, rr, rr2);
    zero_n<N>(pw);
    pw[e2 >> 5] = 1u << (e2 & 31);
    mul(rr, rr, pw);
    copy_n<N>(out, rr);
  }
};

#if defined(__CUDA_ARCH__) && !defined(ZKA_NO_PTX_MUL)
namespace ptx {
template <class F>
static __device__ __noinline__ V8 cios8_mul_fn(V8 a, V8 b) {
  V8 r;
  Field<F>::mul_generic(r.v, a.v, b.v);
  return r;
}
}  // namespace ptx
#endif

using P256p = Field<FpP256>;
using P256n = Field<FnP256>;
using Tomp = Field<FpTom>;
using Tomq = Field<FpP256>;  // tomEdwards256 scalar field == P-256 base field (war256.order is the same prime)
using Warp = Field<FpWar>;

// ------------------------------------------------------------------------------------
// Big-endian byte <-> limb conversion (reference toBytes/fromBytes, big.ts:121-168)
// ------------------------------------------------------------------------------------
template <int N>
ZK_HD void limbs_from_be(uint32_t* r, const uint8_t* b, int nbytes) {
#pragma unroll
  for (int i = 0; i < N; i++) r[i] = 0;
  for (int k = 0; k < nbytes; k++) {
    int pos = nbytes - 1 - k;  // byte significance
    if ((pos >> 2) < N) r[pos >> 2] |= (uint32_t)b[k] << (8 * (pos & 3));
  }
}
template <int N>
ZK_HD void limbs_to_be(uint8_t* b, const uint32_t* a, int nbytes) {
#pragma unroll
  for (int k = 0; k < nbytes; k++) {
    int pos = nbytes - 1 - k;
    b[k] = ((pos >> 2) < N) ? (uint8_t)(a[pos >> 2] >> (8 * (pos & 3))) : 0;
  }
}
// a < m (canonical compare of raw limbs)
template <int N>
ZK_HD bool lt_n(const uint32_t* a, const uint32_t* m) {
#pragma unroll
  for (int i = N - 1; i >= 0; i--) {
    if (a[i] < m[i]) return true;
    if (a[i] > m[i]) return false;
  }
  return false;
}
template <class F>
ZK_HD bool lt_p(const uint32_t* a) {
  return !geq_p<F>(a);
}
// reduce a raw 256-bit integer mod the field prime (inputs < 2^256 < 2p for all our moduli)
template <class F>
ZK_HD void reduce_once(uint32_t* a) {
  uint32_t t[8];
  uint32_t br = sub_p<F>(t, a);
  csel_n<8>(a, br == 0, t, a);
}

}  // namespace zk
