// zk_curves.cuh — group law for P-256 and tomEdwards256 on the GPU.
//
// P-256: homogeneous projective (X:Y:Z), complete a=-3 formulas of Renes-Costello-Batina
//   2015 (Alg. 4 add, Alg. 5 mixed add, Alg. 6 double) — the same formulas the reference
//   uses (/root/reference/src/curves/weier.ts:133-230), on Montgomery residues — wherever
//   arbitrary points meet.  The positional fixed-base walks (accum_fixed) accumulate in
//   Jacobian coordinates with the incomplete mixed addition madd-2007-bl (7M + 4S), whose
//   three exceptional inputs (identity accumulator, P + P, P + (-P)) are tested for and
//   handled exactly; the doubling chains use Jacobian dbl-2001-b.  The device squaring of
//   p256.p is a 36-product multiplier of its own.
// tomEdwards256: the reference works on  a x^2 + y^2 = 1 + d x^2 y^2  with Hisil et al.
//   extended coordinates (/root/reference/src/curves/edwards.ts:141-183).  Here every point
//   is moved once to the isomorphic curve  x'^2 + y^2 = 1 + d' x'^2 y'^2  (x' = sqrt(a) x,
//   d' = d/a; a is a square, d a non-square, so the unified addition stays complete) which
//   saves the multiplication by `a` in every addition; x is mapped back when a point is
//   normalised.  Only affine bytes (toBytes) are observable, so results are bit-identical.
#pragma once
#include "zk_field.cuh"

namespace zk {

// ------------------------------------------------------------------------------------ P-256
#define WEI_PT P256Pt
#define WEI_AFF P256Aff
#define WEI_JAC P256Jac
#define WEI_F P256p
#define WEI_FN(n) p256_##n
#define WEI_B_MONT ZK_P256_B_MONT
#define WEI_GX_MONT ZK_P256_GX_MONT
#define WEI_GY_MONT ZK_P256_GY_MONT
#include "zk_weier.inc"
#undef WEI_PT
#undef WEI_AFF
#undef WEI_JAC
#undef WEI_F
#undef WEI_FN
#undef WEI_B_MONT
#undef WEI_GX_MONT
#undef WEI_GY_MONT

#if defined(ZKA_PG_WAR256)
// ------------------------------------------------------------------------------------ war256
// The war256 build of the library (-DZKA_PG_WAR256 -> libzkattest_war256.so): ProofGroup = war256
// (/root/reference/src/curves/instances.ts:34-41; a legal SystemParametersList.ProofGroup, zkpAttestList.ts:70).
// The curve is short Weierstrass with a = -3 like P-256, so the group law is the second inclusion of zk_weier.inc;
// the stage tasks keep their names and are written against the small proof-group interface below (PGL limbs, PGp
// field, TomPt / TomPre point types, tom_* operations), which the tomEdwards256 build implements with the Edwards
// image curves and this build with the complete Renes-Costello-Batina formulas.
#define WEI_PT WarPt
#define WEI_AFF WarAff
#define WEI_JAC WarJac
#define WEI_F Warp
#define WEI_FN(n) war_##n
#define WEI_B_MONT ZK_WAR_B_MONT
#define WEI_GX_MONT ZK_WAR_GX_MONT
#define WEI_GY_MONT ZK_WAR_GY_MONT
#include "zk_weier.inc"
#undef WEI_PT
#undef WEI_AFF
#undef WEI_JAC
#undef WEI_F
#undef WEI_FN
#undef WEI_B_MONT
#undef WEI_GX_MONT
#undef WEI_GY_MONT

enum : int { PGL = 8 };        // limbs of a proof-group coordinate
using PGp = Warp;              // coordinate field of the proof group
using FpPG = FpWar;
using TomPt = WarPt;           // homogeneous projective (X : Y : Z)
using TomPre = WarAff;         // affine point: table entry / parsed proof point
using TompMsm = Warp;
using TompCommit = Warp;
ZK_HD void tom_set_identity(TomPt& p) { war_set_identity(p); }
ZK_HD void tom_from_affine(TomPt& p, const uint32_t* x, const uint32_t* y) {
  copy_n<8>(p.x, x);
  copy_n<8>(p.y, y);
  Warp::set_one(p.z);
}
ZK_HD void tom_set_generator(TomPt& p) {
  WarAff g;
  war_set_generator(g);
  war_from_affine(p, g);
}
ZK_HD bool tom_on_curve(const uint32_t* x, const uint32_t* y) { return war_on_curve(x, y); }
ZK_HD void tom_add(TomPt& r, const TomPt& p, const TomPt& q) { war_add(r, p, q); }
template <bool kNeedT, class F = Warp>
ZK_HD void tom_madd(TomPt& r, const TomPt& p, const TomPre& q) { war_madd(r, p, q); }
ZK_HD void tom_dbl(TomPt& r, const TomPt& p) { war_dbl(r, p); }
ZK_HD void tom_neg(TomPt& r, const TomPt& p) {
  copy_n<8>(r.x, p.x);
  Warp::neg(r.y, p.y);
  copy_n<8>(r.z, p.z);
}
ZK_HD void pg_dbl_n(TomPt& p, int c) { war_dbl_n(p, c); }
ZK_HD void pg_pre_neg(TomPre& q) { Warp::neg(q.y, q.y); }                       // -(x, y) = (x, -y)
ZK_HD bool pg_is_identity(const TomPt& p) { return war_is_identity(p); }
ZK_HD void pg_fixed_to_msm(TomPt&) {}   // commitments are already (X : Y : Z) of the curve itself
#else
// ----------------------------------------------------------------------------- tomEdwards256
// Extended coordinates on the a'=1 image curve, lazy Montgomery residues mod tom.p.
struct TomPt {
  uint32_t x[9], y[9], t[9], z[9];
};
// Precomputed affine table entry: (x', y, k = d' x' y), canonical residues (< p).
struct TomPre {
  uint32_t x[9], y[9], k[9];
};

ZK_HD void tom_const(uint32_t* r, int which) {
  constexpr uint32_t sa[9] = ZK_TOM_SQRTA_MONT;
  constexpr uint32_t isa[9] = ZK_TOM_INVSQRTA_MONT;
  constexpr uint32_t d1[9] = ZK_TOM_D1_MONT;
  constexpr uint32_t gx[9] = ZK_TOM_GX1_MONT;
  constexpr uint32_t gy[9] = ZK_TOM_GY_MONT;
  constexpr uint32_t s2[9] = ZK_TOM_SQRTND1_MONT;
  constexpr uint32_t is2[9] = ZK_TOM_INVSQRTND1_MONT;
  constexpr uint32_t dd2[9] = ZK_TOM_2D2_MONT;
  constexpr uint32_t isd[9] = ZK_TOM_INVSQRTND_MONT;
#pragma unroll
  for (int i = 0; i < 9; i++)
    r[i] = which == 0 ? sa[i] : which == 1 ? isa[i] : which == 2 ? d1[i] : which == 3 ? gx[i] : which == 4 ? gy[i]
           : which == 5 ? s2[i] : which == 6 ? is2[i] : which == 7 ? dd2[i] : isd[i];
}
enum { TOM_SQRTA = 0, TOM_INVSQRTA = 1, TOM_D1 = 2, TOM_GX1 = 3, TOM_GY = 4, TOM_SQRTND1 = 5, TOM_INVSQRTND1 = 6,
       TOM_2D2 = 7, TOM_INVSQRTND = 8 };

// ---- second image curve E2: -w^2 + v^2 = 1 + d2 w^2 v^2, (w, v) = (sqrt(-d1) x', 1/y) -------------
// Used ONLY by the prover's fixed-base commitment kernel (all its points lie in the prime-order
// subgroup generated by g, where the a = -1 formulas have no exceptional cases; gen_consts.py).
// Table entry: (v - w, v + w, 2 d2 w v).  Mixed addition "madd-2008-hwcd-3": 7M; a walk's first addition (to the
// identity) is 1M (tom2_from_pre) and its last one, when only the normaliser reads the point, 3M (tom2_madd_end).
// Field with the 258-bit multiplier INLINED at every use (no call, no argument marshalling): for loop bodies
// that contain one mixed addition (7-8 products, ~40 KB of code) and are not unrolled.
struct TompInl : Tomp {
  ZK_HD static void mul(uint32_t* r, const uint32_t* a, const uint32_t* b) {
#if defined(__CUDA_ARCH__) && !defined(ZKA_NO_PTX_MUL)
    ptx::tom_mul_body(r, a, b);
#else
    Tomp::mul(r, a, b);
#endif
  }
  ZK_HD static void sqr(uint32_t* r, const uint32_t* a) { mul(r, a, a); }
};
#if defined(ZKA_COMMIT_INLINE)
using TompCommit = TompInl;
#else
using TompCommit = Tomp;
#endif
#if defined(ZKA_MSM_INLINE)
using TompMsm = TompInl;
#else
using TompMsm = Tomp;
#endif

template <bool kNeedT, class F = Tomp>
ZK_HD void tom2_madd(TomPt& r, const TomPt& p, const TomPre& q) {   // q.x = v-w, q.y = v+w, q.k = 2 d2 w v
  uint32_t A[9], B[9], C[9], D[9], E[9], Fv[9], G[9], H[9];
  F::sub(A, p.y, p.x);
  F::mul(A, A, q.x);
  F::add(B, p.y, p.x);
  F::mul(B, B, q.y);
  F::mul(C, p.t, q.k);
  F::add(D, p.z, p.z);
  F::sub(E, B, A);
  F::sub(Fv, D, C);
  F::add(G, D, C);
  F::add(H, B, A);
  F::mul(r.x, E, Fv);
  F::mul(r.y, G, H);
  if (kNeedT) F::mul(r.t, E, H);
  F::mul(r.z, Fv, G);
}
// First point of a walk that starts at the identity: tom2_madd of (0 : 1 : 0 : 1) and q has E = 2w, F = G = 2, H = 2v,
// so the point is (2E : 2H : E H : 4).  1M instead of 7M.  q.x, q.y < p (table entries and their swap), so
// E = q.y + p - q.x < 2p and X < 4p stay inside the bound of tom2_madd's lazy subtraction.
template <class F = Tomp>
ZK_HD void tom2_from_pre(TomPt& r, const TomPre& q) {
  uint32_t E[9], H[9];
#pragma unroll
  for (int i = 0; i < 9; i++) E[i] = FpTom::p(i);
  add_n<9>(E, E, q.y);
  sub_n<9>(E, E, q.x);
  F::add(H, q.y, q.x);
  F::mul(r.t, E, H);
  F::add(r.x, E, E);
  F::add(r.y, H, H);
  F::set_one(r.z);
  F::add(r.z, r.z, r.z);
  F::add(r.z, r.z, r.z);
}
// Last addition of a walk whose point only goes to TomNormTask{e2 = 1}: the E, F, G, H of tom2_madd, of which the
// point is (E F : G H : E H : F G).  The normaliser needs x' sqrt(-d1) = E / G and y = F / H only, so the four
// products X, Y, T, Z are left out: 3M instead of 7M.  Bounds: E < 10p, F < 12p, G < 6p, H < 4p.
struct TomEfgh {
  uint32_t e[9], f[9], g[9], h[9];
};
template <class F = Tomp>
ZK_HD void tom2_madd_end(TomEfgh& r, const TomPt& p, const TomPre& q) {
  uint32_t A[9], B[9], C[9], D[9];
  F::sub(A, p.y, p.x);
  F::mul(A, A, q.x);
  F::add(B, p.y, p.x);
  F::mul(B, B, q.y);
  F::mul(C, p.t, q.k);
  F::add(D, p.z, p.z);
  F::sub(r.e, B, A);
  F::sub(r.f, D, C);
  F::add(r.g, D, C);
  F::add(r.h, B, A);
}

ZK_HD void tom_set_identity(TomPt& p) {
  zero_n<9>(p.x);
  Tomp::set_one(p.y);
  zero_n<9>(p.t);
  Tomp::set_one(p.z);
}
// from affine image-curve coordinates (x', y) (Montgomery)
ZK_HD void tom_from_affine(TomPt& p, const uint32_t* x1, const uint32_t* y) {
  copy_n<9>(p.x, x1);
  copy_n<9>(p.y, y);
  Tomp::mul(p.t, x1, y);
  Tomp::set_one(p.z);
}
ZK_HD void tom_set_generator(TomPt& p) {
  uint32_t gx[9], gy[9];
  tom_const(gx, TOM_GX1);
  tom_const(gy, TOM_GY);
  tom_from_affine(p, gx, gy);
}
// x'^2 + y^2 == 1 + d' x'^2 y^2   (edwards.ts:52-65 on the image curve, z = 1)
ZK_HD bool tom_on_curve(const uint32_t* x1, const uint32_t* y) {
  using F = Tomp;
  uint32_t xx[9], yy[9], l[9], r[9], d1[9], one[9];
  F::sqr(xx, x1);
  F::sqr(yy, y);
  F::add(l, xx, yy);
  F::mul(r, xx, yy);
  tom_const(d1, TOM_D1);
  F::mul(r, r, d1);
  F::set_one(one);
  F::add(r, r, one);
  // l == r  <=>  (l - r) * 1 / R is 0 or p: one Montgomery product (output < 2p) and two compares instead of
  // two 14-step canonical-reduction ladders (this test runs once per point of every proof in VValidateTask)
  uint32_t d[9], o[9];
  F::sub(d, l, r);               // l + 8p - r, r < 3p
  zero_n<9>(o);
  o[0] = 1;
  F::mul(d, d, o);
  uint32_t nz = 0, np = 0;
#pragma unroll
  for (int i = 0; i < 9; i++) { nz |= d[i]; np |= d[i] ^ FpTom::p(i); }
  return nz == 0 || np == 0;
}

// Hisil et al. 2008 section 3.1 unified addition with a = 1 (edwards.ts:161-183): 9M
ZK_HD void tom_add(TomPt& r, const TomPt& p, const TomPt& q) {
  using F = Tomp;
  uint32_t A[9], B[9], C[9], D[9], E[9], Fv[9], G[9], H[9], d1[9];
  tom_const(d1, TOM_D1);
  F::mul(A, p.x, q.x);
  F::mul(B, p.y, q.y);
  F::mul(C, p.t, q.t);
  F::mul(C, C, d1);
  F::mul(D, p.z, q.z);
  F::add(E, p.x, p.y);
  F::add(H, q.x, q.y);
  F::mul(E, E, H);
  F::sub(E, E, A);
  F::sub(E, E, B);
  F::sub(Fv, D, C);
  F::add(G, D, C);
  F::sub(H, B, A);
  F::mul(r.x, E, Fv);
  F::mul(r.y, G, H);
  F::mul(r.t, E, H);
  F::mul(r.z, Fv, G);
}
// mixed addition with a precomputed entry (Z2 = 1, k = d' x2 y2): 7M (+1M for T3)
template <bool kNeedT, class F = Tomp>
ZK_HD void tom_madd(TomPt& r, const TomPt& p, const TomPre& q) {
  uint32_t A[9], B[9], C[9], E[9], Fv[9], G[9], H[9];
  F::mul(A, p.x, q.x);
  F::mul(B, p.y, q.y);
  F::mul(C, p.t, q.k);
  F::add(E, p.x, p.y);
  F::add(H, q.x, q.y);
  F::mul(E, E, H);
  F::sub(E, E, A);
  F::sub(E, E, B);
  F::sub(Fv, p.z, C);
  F::add(G, p.z, C);
  F::sub(H, B, A);
  F::mul(r.x, E, Fv);
  F::mul(r.y, G, H);
  if (kNeedT) F::mul(r.t, E, H);
  F::mul(r.z, Fv, G);
}
// Hisil et al. 2008 section 3.3 doubling with a = 1 (edwards.ts:141-160): 4M + 4S
ZK_HD void tom_dbl(TomPt& r, const TomPt& p) {
  using F = Tomp;
  uint32_t A[9], B[9], C[9], E[9], G[9], Fv[9], H[9];
  F::sqr(A, p.x);
  F::sqr(B, p.y);
  F::sqr(C, p.z);
  F::add(C, C, C);
  F::add(E, p.x, p.y);
  F::sqr(E, E);
  F::sub(E, E, A);
  F::sub(E, E, B);
  F::add(G, A, B);   // D + B with D = a'A = A
  F::sub(Fv, G, C);
  F::sub(H, A, B);   // D - B
  F::mul(r.x, E, Fv);
  F::mul(r.y, G, H);
  F::mul(r.t, E, H);
  F::mul(r.z, Fv, G);
}
ZK_HD void tom_neg(TomPt& r, const TomPt& p) {
  Tomp::neg(r.x, p.x);
  copy_n<9>(r.y, p.y);
  Tomp::neg(r.t, p.t);
  copy_n<9>(r.z, p.z);
}


enum : int { PGL = 9 };        // limbs of a proof-group coordinate
using PGp = Tomp;              // coordinate field of the proof group
using FpPG = FpTom;
ZK_HD void pg_dbl_n(TomPt& p, int c) {
  for (int i = 0; i < c; i++) tom_dbl(p, p);
}
ZK_HD void pg_pre_neg(TomPre& q) {   // -(x, y) = (-x, y); k = d x y changes sign too
  Tomp::neg(q.x, q.x);
  Tomp::neg(q.k, q.k);
}
// identity <=> X == 0 and Y == Z (edwards.ts:117-125 in projective form)
ZK_HD bool pg_is_identity(const TomPt& p) { return Tomp::is_zero(p.x) && Tomp::eq(p.y, p.z); }
// A fixed-base commitment comes out of the commitment kernels on the a = -1 image curve E2 as (W : V : Z) with
// x' = W / (Z sqrt(-d1)), y = Z / V.  Same point in E1 extended coordinates with Z' = Z V:
//   X = c W V,  Y = Z^2,  T = X Y / Z' = c W Z,   c = 1/sqrt(-d1).
ZK_HD void pg_fixed_to_msm(TomPt& f) {
  uint32_t cw[9], X[9], Y[9], Tt[9], Zp[9], c1[9];
  tom_const(c1, TOM_INVSQRTND1);
  Tomp::mul(cw, f.x, c1);
  Tomp::mul(X, cw, f.y);
  Tomp::sqr(Y, f.z);
  Tomp::mul(Tt, cw, f.z);
  Tomp::mul(Zp, f.z, f.y);
  copy_n<9>(f.x, X); copy_n<9>(f.y, Y); copy_n<9>(f.t, Tt); copy_n<9>(f.z, Zp);
}
#endif   // ZKA_PG_WAR256

}  // namespace zk
