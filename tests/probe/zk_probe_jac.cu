// zk_probe_jac.cu — test-only probe of the P-256 squaring, the Jacobian + affine mixed addition and the Jacobian
// fixed-base walk (tests/test_p256_jacobian.py).  It is zk_probe.cu (all of its entry points and helpers) plus the
// entry points below, built the same two ways: nvcc for sm_90a (libzkprobe_jac.so) and g++ -DZKA_HOSTSIM
// (libzkprobe_jac_host.so).  Never loaded by the product.  Same conventions: raw little-endian 32-bit limbs, 9 words
// per field element, 0 / -1 (bad argument) / -2 (CUDA error) returns, no asserts or traps in device code.
#include "zk_probe.cu"

namespace {

// out[i] = Field<F>::sqr(a[i]) in field 0 p256.p, 1 p256.n, 2 tom.p, 3 war.p
struct SqrTask {
  int field;
  const uint32_t* a;
  uint32_t* out;
  template <class F>
  ZK_HD void run(const uint32_t* x, uint32_t* r) const {
    uint32_t v[F::N], z[F::N];
    copy_n<F::N>(v, x);
    Field<F>::sqr(z, v);
    copy_n<F::N>(r, z);
  }
  ZK_HD void operator()(int i) const {
    const size_t o = (size_t)i * W;
    uint32_t r[W] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
    if (field == 0) run<FpP256>(a + o, r);
    else if (field == 1) run<FnP256>(a + o, r);
    else if (field == 2) run<FpTom>(a + o, r);
    else run<FpWar>(a + o, r);
    for (int k = 0; k < W; k++) out[o + k] = r[k];
  }
};

// production sqr(a) against mul_generic(a, a) on hashed operands (draw_operand), plus the output bound
struct SqrDiffTask {
  int field, bound_bits, per;
  uint64_t seed, count;
  uint32_t* mismatches;   // [1]
  uint32_t* bad;          // [16][2][W]: a, production output of the first mismatches
  template <class F>
  ZK_HD void run(int t) const {
    constexpr int N = F::N;
    uint32_t bd[N + 1], lim[N + 1];
    bound_of<F>(bd, bound_bits);
    bound_of<F>(lim, F::kLazy ? 1 : 0);
    for (int j = 0; j < per; j++) {
      const uint64_t idx = (uint64_t)t * (uint64_t)per + (uint64_t)j;
      if (idx >= count) return;
      uint32_t a[N], r[N], g[N];
      draw_operand<F>(a, seed, idx, bd);
      Field<F>::sqr(r, a);
      Field<F>::mul_generic(g, a, a);
      if (!eq_n<N>(r, g) || !lt_wide<F>(r, lim)) {
        const uint32_t k = zk_atomic_add(mismatches, 1u);
        if (k < 16) {
          uint32_t* o = bad + (size_t)k * 2 * W;
          for (int i = 0; i < W; i++) {
            o[i] = i < N ? a[i] : 0u;
            o[W + i] = i < N ? r[i] : 0u;
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

// r = p + q, p Jacobian (X, Y, Z), q affine (x, y): rows of [X, Y, Z, x, y] x 8 words in, [X, Y, Z] x 8 out
struct JacMaddTask {
  const uint32_t* in;
  uint32_t* out;
  ZK_HD void operator()(int i) const {
    const uint32_t* s = in + (size_t)i * 40;
    P256Jac p, r;
    P256Aff q;
    copy_n<8>(p.x, s); copy_n<8>(p.y, s + 8); copy_n<8>(p.z, s + 16);
    copy_n<8>(q.x, s + 24); copy_n<8>(q.y, s + 32);
    p256_jac_madd(r, p, q);
    uint32_t* o = out + (size_t)i * 24;
    copy_n<8>(o, r.x); copy_n<8>(o + 8, r.y); copy_n<8>(o + 16, r.z);
  }
};

// acc += k * base on a caller's table, through p256_accum_fixed_jac (jac = 1, Jacobian accumulator) or
// p256_accum_fixed (jac = 0, homogeneous)
struct AccumTask {
  int jac, w;
  const uint32_t* tab;       // [fb_windows(w)][fb_entries(w)][16] affine Montgomery entries
  const uint32_t* scalars;   // [count][8]
  const uint32_t* acc_in;    // [count][24]  X, Y, Z
  uint32_t* out;             // [count][24]  the same coordinates as the input
  ZK_HD void operator()(int i) const {
    const uint32_t* a = acc_in + (size_t)i * 24;
    uint32_t* o = out + (size_t)i * 24;
    if (jac) {
      P256Jac acc;
      copy_n<8>(acc.x, a); copy_n<8>(acc.y, a + 8); copy_n<8>(acc.z, a + 16);
      p256_accum_fixed_jac(acc, tab, scalars + (size_t)i * 8, w);
      copy_n<8>(o, acc.x); copy_n<8>(o + 8, acc.y); copy_n<8>(o + 16, acc.z);
    } else {
      P256Pt acc;
      copy_n<8>(acc.x, a); copy_n<8>(acc.y, a + 8); copy_n<8>(acc.z, a + 16);
      p256_accum_fixed(acc, tab, scalars + (size_t)i * 8, w);
      copy_n<8>(o, acc.x); copy_n<8>(o + 8, acc.y); copy_n<8>(o + 16, acc.z);
    }
  }
};

}  // namespace

extern "C" {

int probe_sqr(int field, int count, const uint32_t* a, uint32_t* out) {
  if (field < 0 || field > 3 || count < 0) return -1;
  return guarded([&] {
    const size_t bytes = (size_t)count * W * 4;
    Buf da(bytes), dout(bytes);
    Stream st;
    copy_h2d(st, da.p, a, bytes);
    launch(st, count, SqrTask{field, da.as<uint32_t>(), dout.as<uint32_t>()});
    copy_d2h(st, out, dout.p, bytes);
    sync(st);
    return 0;
  });
}

// `count` squarings of hashed operands below 2^bound_bits * p (`per` per thread); *mismatches and bad[16][2][9]
int probe_sqr_diff(int field, uint64_t seed, uint64_t count, int bound_bits, int per, uint32_t* mismatches,
                   uint32_t* bad) {
  if (field < 0 || field > 3 || per < 1 || bound_bits < 0 || bound_bits > 13) return -1;
  const uint64_t threads = (count + (uint64_t)per - 1) / (uint64_t)per;
  if (threads > 0x7fffffffull) return -1;
  return guarded([&] {
    const size_t bb = (size_t)16 * 2 * W * 4;
    Buf dm(4), dbad(bb);
    Stream st;
    dev_memset(st, dm.p, 0, 4);
    dev_memset(st, dbad.p, 0, bb);
    launch(st, (long long)threads, SqrDiffTask{field, bound_bits, per, seed, count, dm.as<uint32_t>(), dbad.as<uint32_t>()});
    copy_d2h(st, mismatches, dm.p, 4);
    copy_d2h(st, bad, dbad.p, bb);
    sync(st);
    return 0;
  });
}

int probe_jac_madd(int count, const uint32_t* in, uint32_t* out) {
  if (count < 0) return -1;
  return guarded([&] {
    const size_t ib = (size_t)count * 40 * 4, ob = (size_t)count * 24 * 4;
    Buf di(ib), dout(ob);
    Stream st;
    copy_h2d(st, di.p, in, ib);
    launch(st, count, JacMaddTask{di.as<uint32_t>(), dout.as<uint32_t>()});
    copy_d2h(st, out, dout.p, ob);
    sync(st);
    return 0;
  });
}

// out[i] = acc_in[i] + scalars[i] * base on the caller's table; 2 <= w <= 24
int probe_p256_accum(int jac, int w, int count, const uint32_t* tab, const uint32_t* scalars, const uint32_t* acc_in,
                     uint32_t* out) {
  if (w < 2 || w > 24 || count < 0) return -1;
  return guarded([&] {
    const size_t tb = (size_t)fb_windows(w) * fb_entries(w) * 16 * 4, sb = (size_t)count * 32, ab = (size_t)count * 96;
    Buf dt(tb), ds(sb), da(ab), dout(ab);
    Stream st;
    copy_h2d(st, dt.p, tab, tb);
    copy_h2d(st, ds.p, scalars, sb);
    copy_h2d(st, da.p, acc_in, ab);
    launch(st, count, AccumTask{jac, w, dt.as<uint32_t>(), ds.as<uint32_t>(), da.as<uint32_t>(), dout.as<uint32_t>()});
    copy_d2h(st, out, dout.p, ab);
    sync(st);
    return 0;
  });
}

}  // extern "C"
