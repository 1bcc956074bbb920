// zk_probe.cu — test-only arithmetic probe: the field operations and scalar recoders of the library on raw operands.
//
// Built twice, like the host simulator: nvcc for sm_90a (libzkprobe.so, the production device code including the PTX
// multipliers) and g++ with -DZKA_HOSTSIM (libzkprobe_host.so).  Never loaded by the product.  Inputs and outputs are
// little-endian 32-bit limbs, 9 words per element for every field; nothing is converted to Montgomery form, reduced
// or byte-encoded on the way in or out, so an operand can be anywhere in an operation's documented domain.
// Every entry point returns 0, or -1 for an unknown field / op / kind, or -2 for a CUDA error.  Device code never
// asserts or traps: the differential check reports through a counter.
#include "zk_field.cuh"
#include "zk_curves.cuh"
#include "zk_ops.cuh"
#include "zk_verify_agg.cuh"
#include "zk_launch.cuh"

using namespace zk;

namespace {

enum { W = 9 };                 // words per element in the probe's buffers
enum { DIGIT_ROW = 132 };       // ints per scalar in probe_digits: digits, then [129..131] = aux values

enum Op { OP_MUL, OP_MUL_GENERIC, OP_MUL_INL, OP_ADD, OP_SUB, OP_NEG, OP_REDUCE, OP_FROM_MONT, OP_IS_ZERO, OP_EQ,
          OP_INV, OP_COUNT };

template <class F>
ZK_HD bool field_op(int op, uint32_t* r, const uint32_t* a, const uint32_t* b) {
  constexpr int N = F::N;
  using Fd = Field<F>;
  uint32_t x[N], y[N], z[N];
  copy_n<N>(x, a);
  copy_n<N>(y, b);
  zero_n<N>(z);
  switch (op) {
    case OP_MUL: Fd::mul(z, x, y); break;
    case OP_MUL_GENERIC: Fd::mul_generic(z, x, y); break;
    case OP_MUL_INL:   // tom.p only
      if constexpr (same_t<F, FpTom>::value) TompInl::mul(z, x, y);
      else return false;
      break;
    case OP_ADD: Fd::add(z, x, y); break;
    case OP_SUB: Fd::sub(z, x, y); break;
    case OP_NEG: Fd::neg(z, x); break;
    case OP_REDUCE: copy_n<N>(z, x); Fd::reduce(z); break;
    case OP_FROM_MONT: Fd::from_mont(z, x); break;
    case OP_IS_ZERO: z[0] = Fd::is_zero(x) ? 1u : 0u; break;
    case OP_EQ: z[0] = Fd::eq(x, y) ? 1u : 0u; break;
    case OP_INV: Fd::inv(z, x); break;
    default: return false;
  }
  copy_n<N>(r, z);
  return true;
}

struct FieldTask {
  int field, op;
  const uint32_t *a, *b;
  uint32_t* out;
  ZK_HD void operator()(int i) const {
    const size_t o = (size_t)i * W;
    uint32_t r[W] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
    if (field == 0) field_op<FpP256>(op, r, a + o, b + o);
    else if (field == 1) field_op<FnP256>(op, r, a + o, b + o);
    else if (field == 2) field_op<FpTom>(op, r, a + o, b + o);
    else field_op<FpWar>(op, r, a + o, b + o);
    for (int k = 0; k < W; k++) out[o + k] = r[k];
  }
};

// ---- differential check: production mul against the generic CIOS on hashed operands --------------------------------
ZK_HD uint64_t mix64(uint64_t x) {   // splitmix64 finaliser
  x += 0x9e3779b97f4a7c15ull;
  x = (x ^ (x >> 30)) * 0xbf58476d1ce4e5b9ull;
  x = (x ^ (x >> 27)) * 0x94d049bb133111ebull;
  return x ^ (x >> 31);
}
// bound = 2^bound_bits * p, in N+1 limbs
template <class F>
ZK_HD void bound_of(uint32_t* bd, int bound_bits) {
  constexpr int N = F::N;
  bd[N] = 0;
  for (int i = 0; i < N; i++) bd[i] = F::p(i);
  for (int s = 0; s < bound_bits; s++) {
    uint32_t c = 0;
    for (int i = 0; i <= N; i++) { const uint32_t v = bd[i]; bd[i] = (v << 1) | c; c = v >> 31; }
  }
}
// an operand in [0, bound): random bit length, all-ones / zero limb patterns, or just below the bound
template <class F>
ZK_HD void draw_operand(uint32_t* x, uint64_t seed, uint64_t idx, const uint32_t* bd) {
  constexpr int N = F::N;
  uint64_t h = mix64(seed ^ mix64(idx));
  int top = N * 32;
  while (top > 0 && !((bd[(top - 1) >> 5] >> ((top - 1) & 31)) & 1u)) top--;   // bit length of the bound
  const int mode = (int)(h & 3);
  const int len = mode == 1 ? 1 + (int)((h >> 8) % (uint64_t)top) : top;
  for (int i = 0; i < N; i++) {
    h = mix64(h + (uint64_t)i);
    uint32_t v = (uint32_t)h;
    if (mode == 2) {
      const int pat = (int)((h >> 32) & 3);
      v = pat == 0 ? 0u : pat == 1 ? 0xffffffffu : pat == 2 ? (uint32_t)(h >> 40) : v;
    }
    x[i] = v;
  }
  for (int i = 0; i < N; i++) {   // keep bits [0, len)
    const int lo = 32 * i;
    if (lo >= len) x[i] = 0;
    else if (len - lo < 32) x[i] &= (1u << (len - lo)) - 1u;
  }
  if (mode == 3) {                // bound - 1 - small
    uint32_t s[N];
    zero_n<N>(s);
    s[0] = 1u + (uint32_t)((h >> 32) & 0xffff);
    sub_n<N>(x, bd, s);
    return;
  }
  uint32_t t[N];   // x < 2^top <= 2 bound: one conditional subtraction
  const uint32_t br = sub_n<N>(t, x, bd);
  const bool ge = br == 0 && bd[N] == 0;
  csel_n<N>(x, ge, t, x);
}
template <class F>
ZK_HD bool lt_wide(const uint32_t* a, const uint32_t* bd) {   // a (N limbs) < bd (N+1 limbs)
  if (bd[F::N]) return true;
  return lt_n<F::N>(a, bd);
}

struct MulDiffTask {
  int field, bound_bits, per;
  uint64_t seed, count;
  uint32_t* mismatches;   // [1]
  uint32_t* bad;          // [16][3][W]: a, b, production output of the first mismatches
  template <class F>
  ZK_HD void run(int t) const {
    constexpr int N = F::N;
    uint32_t bd[N + 1], lim[N + 1];
    bound_of<F>(bd, bound_bits);
    bound_of<F>(lim, F::kLazy ? 1 : 0);   // output bound: 2p lazy, p strict
    for (int j = 0; j < per; j++) {
      const uint64_t idx = (uint64_t)t * (uint64_t)per + (uint64_t)j;
      if (idx >= count) return;
      uint32_t a[N], b[N], r[N], g[N];
      draw_operand<F>(a, seed, 2 * idx, bd);
      draw_operand<F>(b, seed, 2 * idx + 1, bd);
      Field<F>::mul(r, a, b);
      Field<F>::mul_generic(g, a, b);
      if (!eq_n<N>(r, g) || !lt_wide<F>(r, lim)) {
        const uint32_t k = zk_atomic_add(mismatches, 1u);
        if (k < 16) {
          uint32_t* o = bad + (size_t)k * 3 * W;
          for (int i = 0; i < W; i++) {
            o[i] = i < N ? a[i] : 0u;
            o[W + i] = i < N ? b[i] : 0u;
            o[2 * W + i] = i < N ? r[i] : 0u;
          }
        }
      }
    }
  }
  ZK_HD void operator()(int t) const {
    if (field == 0) run<FpP256>(t);
    else if (field == 1) run<FnP256>(t);
    else if (field == 2) run<FpTom>(t);
    else run<FpWar>(t);
  }
};

// ---- scalar recoders ------------------------------------------------------------------------------------------------
enum Kind { K_SIGNED, K_MSM6, K_MSM4, K_AGG };
struct DigitTask {
  int kind, w;
  AggDigits D;
  const uint32_t* scalars;   // [count][8]
  int32_t* out;              // [count][DIGIT_ROW] (agg: [count][2][DIGIT_ROW], digits then buckets)
  ZK_HD void operator()(int i) const {
    const uint32_t* k = scalars + (size_t)i * 8;
    int32_t* o = out + (size_t)i * (kind == K_AGG ? 2 : 1) * DIGIT_ROW;
    if (kind == K_SIGNED) {
      uint32_t carry = 0;
      const int nw = fb_windows(w);
      for (int j = 0; j < nw; j++) {
        bool neg;
        const uint32_t d = signed_digit(k, j, w, carry, neg);
        o[j] = neg ? -(int32_t)d : (int32_t)d;
      }
      o[DIGIT_ROW - 1] = (int32_t)carry;
    } else if (kind == K_MSM6 || kind == K_MSM4) {
      const int nw = kind == K_MSM6 ? MSM_NWIN : MSM_NWIN_N;
      for (int j = 0; j < nw; j++) {
        bool neg;
        const uint32_t d = kind == K_MSM6 ? msm_digit6(k, j, neg) : msm_digit4(k, j, neg);
        o[j] = neg ? -(int32_t)d : (int32_t)d;
      }
    } else {
      uint32_t kp[10];
      agg_kp(kp, k, D);
      for (int j = 0; j < D.nwin; j++) {
        const int d = agg_digit(kp, j, D.c);
        o[j] = d;
        o[DIGIT_ROW + j] = d ? (int32_t)agg_bucket(D, j, d < 0 ? -d : d, i) : 0;
      }
    }
  }
};

// ---- group law: points as raw Montgomery limbs, [X, Y, T|-, Z|-] in 9-word slots -------------------------------------
enum GroupOp { G_P256_ADD, G_P256_MADD, G_P256_DBL, G_P256_JAC_DBL, G_TOM_ADD, G_TOM_MADD, G_TOM_DBL, G_TOM_CONST,
               G_COUNT };
struct GroupTask {
  int op;
  const uint32_t* in;   // [count][2][4][W]: P, Q (Q of a mixed addition: affine x, y; tom: x', y, k = d' x' y)
  uint32_t* out;        // [count][4][W]
  ZK_HD void operator()(int i) const {
    const uint32_t* p = in + (size_t)i * 8 * W;
    const uint32_t* q = p + 4 * W;
    uint32_t* o = out + (size_t)i * 4 * W;
    if (op <= G_P256_JAC_DBL) {
      P256Pt a, b, r;
      copy_n<8>(a.x, p); copy_n<8>(a.y, p + W); copy_n<8>(a.z, p + 3 * W);
      copy_n<8>(b.x, q); copy_n<8>(b.y, q + W); copy_n<8>(b.z, q + 3 * W);
      if (op == G_P256_ADD) p256_add(r, a, b);
      else if (op == G_P256_DBL) p256_dbl(r, a);
      else if (op == G_P256_MADD) {
        P256Aff qa;
        copy_n<8>(qa.x, q); copy_n<8>(qa.y, q + W);
        p256_madd(r, a, qa);
      } else {
        P256Jac j, jr;
        copy_n<8>(j.x, a.x); copy_n<8>(j.y, a.y); copy_n<8>(j.z, a.z);
        p256_jac_dbl(jr, j);
        copy_n<8>(r.x, jr.x); copy_n<8>(r.y, jr.y); copy_n<8>(r.z, jr.z);
      }
      copy_n<8>(o, r.x); copy_n<8>(o + W, r.y); copy_n<8>(o + 3 * W, r.z);
    } else if (op == G_TOM_CONST) {
      tom_const(o, (int)p[0]);
    } else {
      TomPt a, b, r;
      copy_n<9>(a.x, p); copy_n<9>(a.y, p + W); copy_n<9>(a.t, p + 2 * W); copy_n<9>(a.z, p + 3 * W);
      copy_n<9>(b.x, q); copy_n<9>(b.y, q + W); copy_n<9>(b.t, q + 2 * W); copy_n<9>(b.z, q + 3 * W);
      if (op == G_TOM_ADD) tom_add(r, a, b);
      else if (op == G_TOM_DBL) tom_dbl(r, a);
      else {
        TomPre e;
        copy_n<9>(e.x, b.x); copy_n<9>(e.y, b.y); copy_n<9>(e.k, b.t);
        tom_madd<true>(r, a, e);
      }
      copy_n<9>(o, r.x); copy_n<9>(o + W, r.y); copy_n<9>(o + 2 * W, r.t); copy_n<9>(o + 3 * W, r.z);
    }
  }
};

// ---- host side ------------------------------------------------------------------------------------------------------
struct Buf {
  void* p = nullptr;
  explicit Buf(size_t n) : p(dev_alloc(n)) {}
  ~Buf() { dev_free(p); }
  template <class T> T* as() const { return static_cast<T*>(p); }
};

template <class Fn>
int guarded(Fn&& fn) {
  try {
    return fn();
  } catch (const std::exception&) {
    return -2;
  }
}

}  // namespace

extern "C" {

// out[i] = op(a[i], b[i]) in field 0 p256.p, 1 p256.n, 2 tom.p, 3 war.p; 9 words per element
// (is_zero / eq: out[i][0] = 0 or 1).  Ops: see enum Op.
int probe_field(int field, int op, int count, const uint32_t* a, const uint32_t* b, uint32_t* out) {
  if (field < 0 || field > 3 || op < 0 || op >= OP_COUNT || count < 0) return -1;
  if (op == OP_MUL_INL && field != 2) return -1;
  return guarded([&] {
    const size_t bytes = (size_t)count * W * 4;
    Buf da(bytes), db(bytes), dout(bytes);
    Stream st;
    copy_h2d(st, da.p, a, bytes);
    copy_h2d(st, db.p, b, bytes);
    launch(st, count, FieldTask{field, op, da.as<uint32_t>(), db.as<uint32_t>(), dout.as<uint32_t>()});
    copy_d2h(st, out, dout.p, bytes);
    sync(st);
    return 0;
  });
}

// `count` products of hashed operands below 2^bound_bits * p (`per` per thread): production mul against mul_generic,
// plus the output bound (< 2p for tom.p, < p otherwise).  Returns the number of mismatches in *mismatches and the
// operands and production output of the first 16 in bad[16][3][9].
int probe_mul_diff(int field, uint64_t seed, uint64_t count, int bound_bits, int per, uint32_t* mismatches,
                   uint32_t* bad) {
  if (field < 0 || field > 3 || per < 1 || bound_bits < 0 || bound_bits > 13) return -1;
  const uint64_t threads = (count + (uint64_t)per - 1) / (uint64_t)per;
  if (threads > 0x7fffffffull) return -1;
  return guarded([&] {
    Buf dm(4), dbad((size_t)16 * 3 * W * 4);
    Stream st;
    dev_memset(st, dm.p, 0, 4);
    dev_memset(st, dbad.p, 0, (size_t)16 * 3 * W * 4);
    launch(st, (long long)threads, MulDiffTask{field, bound_bits, per, seed, count, dm.as<uint32_t>(), dbad.as<uint32_t>()});
    copy_d2h(st, mismatches, dm.p, 4);
    copy_d2h(st, bad, dbad.p, (size_t)16 * 3 * W * 4);
    sync(st);
    return 0;
  });
}

// digits of each 8-limb scalar: kind 0 signed_digit (w = 2..24, fb_windows(w) digits, final carry at [131]),
// 1 msm_digit6 (MSM_NWIN digits), 2 msm_digit4 (MSM_NWIN_N digits), 3 the aggregate MSM's digits for c = w (agg_plan):
// rows of 2 x 132 ints, digits then bucket indices (slot = scalar index); aux[0..3] = c, nwin, nb, top_shift.
int probe_digits(int kind, int w, int count, const uint32_t* scalars, int32_t* out, int32_t* aux) {
  if (kind < 0 || kind > 3 || count < 0) return -1;
  if (kind == K_SIGNED && (w < 2 || w > 24)) return -1;
  if (kind == K_AGG && (w < 4 || w > 16)) return -1;
  const AggDigits D = agg_plan(1.0, kind == K_AGG ? w : 4).D;
  if (aux) { aux[0] = D.c; aux[1] = D.nwin; aux[2] = D.nb; aux[3] = D.top_shift; }
  return guarded([&] {
    const size_t row = (size_t)(kind == K_AGG ? 2 : 1) * DIGIT_ROW * 4;
    Buf ds((size_t)count * 32), dout((size_t)count * row);
    Stream st;
    copy_h2d(st, ds.p, scalars, (size_t)count * 32);
    dev_memset(st, dout.p, 0, (size_t)count * row);
    launch(st, count, DigitTask{kind, w, D, ds.as<uint32_t>(), dout.as<int32_t>()});
    copy_d2h(st, out, dout.p, (size_t)count * row);
    sync(st);
    return 0;
  });
}

// group law on raw Montgomery coordinates (see GroupOp / GroupTask): P-256 add / madd / dbl (homogeneous) and the
// Jacobian doubling of the aggregate MSM's Horner step, tomEdwards256 E1 add / madd / dbl (extended, a' = 1 image),
// and tom_const(which) for the image-curve constants.
int probe_group(int op, int count, const uint32_t* in, uint32_t* out) {
  if (op < 0 || op >= G_COUNT || count < 0) return -1;
  return guarded([&] {
    const size_t ib = (size_t)count * 8 * W * 4, ob = (size_t)count * 4 * W * 4;
    Buf di(ib), dout(ob);
    Stream st;
    copy_h2d(st, di.p, in, ib);
    dev_memset(st, dout.p, 0, ob);
    launch(st, count, GroupTask{op, di.as<uint32_t>(), dout.as<uint32_t>()});
    copy_d2h(st, out, dout.p, ob);
    sync(st);
    return 0;
  });
}

}  // extern "C"
