// zk_sigma.cuh — the sigma-protocol layer of a PointAddProof, shared by the prover and both verifiers.
//
//   /root/reference/src/commit/equality.ts:60-116  EqualityProof: prove, aggregateEquality (2 relations)
//   /root/reference/src/commit/mult.ts:93-175      MultProof: prove, aggregateMult (5 relations)
//   /root/reference/src/exp/pointAdd.ts:92-259     PointAddProof: four MultProofs and two EqualityProofs
//
// One place each for: the point and scalar encodings (the proof group's and P-256's), which commitments make up the
// statement of every sub-proof (the wiring), the five derived commitments, the prover steps of a MultProof and an
// EqualityProof (openings and responses), the deserialisation checks of a proof body, and the relation folds of the
// verifiers.
#pragma once
#include "zk_ops.cuh"

namespace zk {

// ---- encodings of the proof group --------------------------------------------------------------------------------
#if defined(ZKA_PG_WAR256)
// parse a war256 point encoding (SEC1 uncompressed, weier.ts:74-89: 0x04 tag, on curve) -> affine Montgomery; returns
// validity.  Like p256_parse, and like the reference (no range check; the curve equation is checked mod p), a
// coordinate in [p, 2^256) stands for its residue.  (The identity has no 65-byte encoding in a proof slot: tag 0x00 is
// malformed here.)
ZK_HD bool tom_parse(uint32_t* xm, uint32_t* ym, const uint8_t* b) {
  uint32_t x[8], y[8];
  limbs_from_be<8>(x, b + 1, 32);
  limbs_from_be<8>(y, b + 33, 32);
  const bool ok = b[0] == 0x04;
  reduce_once<FpWar>(x);
  reduce_once<FpWar>(y);
  Warp::to_mont(xm, x);
  Warp::to_mont(ym, y);
  return ok && war_on_curve(xm, ym);
}
#else
// parse a tomEdwards256 point encoding -> image-curve affine Montgomery; returns validity
// (edwards.ts:70-86: 0x04 tag, coordinates < p, on curve)
ZK_HD bool tom_parse(uint32_t* xm, uint32_t* ym, const uint8_t* b) {
  uint32_t x[9], y[9], sa[9];
  limbs_from_be<9>(x, b + 1, 33);
  limbs_from_be<9>(y, b + 34, 33);
  bool ok = (b[0] == 0x04) && lt_p<FpTom>(x) && lt_p<FpTom>(y);
  Tomp::to_mont(xm, x);
  Tomp::to_mont(ym, y);
  tom_const(sa, TOM_SQRTA);
  Tomp::mul(xm, xm, sa);
  return ok && tom_on_curve(xm, ym);
}
#endif
ZK_HD bool wscalar_parse(uint32_t* r, const uint8_t* b) {   // WS bytes (33 tomEdwards256 / 32 war256), mod the group order
  limbs_from_be<8>(r, b + (WS - 32), 32);
  return (WS == 32 || b[0] == 0) && lt_p<FpP256>(r);
}
// P-256 point encoding -> affine Montgomery; returns validity.  65 zero bytes are the identity: inf is set, a holds the
// generator and the encoding counts as valid (each caller decides whether it accepts the identity).  Otherwise the tag
// must be 0x04 and the point on the curve; as in weier.ts:74-89 a coordinate in [p, 2^256) stands for its residue.  An
// invalid encoding leaves its reduced coordinates in a.
ZK_HD bool p256_parse(P256Aff& a, bool& inf, const uint8_t* b) {
  uint32_t x[8], y[8];
  limbs_from_be<8>(x, b + 1, 32);
  limbs_from_be<8>(y, b + 33, 32);
  inf = (b[0] == 0) && is_zero_n<8>(x) && is_zero_n<8>(y);
  if (inf) { p256_set_generator(a); return true; }
  reduce_once<FpP256>(x);
  reduce_once<FpP256>(y);
  P256p::to_mont(a.x, x);
  P256p::to_mont(a.y, y);
  return b[0] == 0x04 && p256_on_curve(a.x, a.y);
}
// scalar encodings (group.ts:62-66 deserializeScalar: value < order)
ZK_HD bool nscalar_parse(uint32_t* r, const uint8_t* b) {   // 32 bytes, mod p256.n
  limbs_from_be<8>(r, b, 32);
  return lt_p<FnP256>(r);
}
// a verifier draw (Relation.drain): 32 bytes below p256.n (nist) or the proof group's order
ZK_HD bool vdraw(uint32_t* r, const uint8_t* p, bool nist) {
  limbs_from_be<8>(r, p, 32);
  return nist ? lt_p<FnP256>(r) : lt_p<FpP256>(r);
}

// ---- wiring of a PointAddProof ------------------------------------------------------------------------------------
// The commitments its sub-proofs talk about.  C8, C10, C11, C13 are its own points, g is ProofGroup.g (C14,
// pointAdd.ts:144), and C7, C9, C12, Cint, Cint2 are derived from the statement C1..C6 (point_add_derived).
enum : int { PA_C7, PA_C8, PA_G, PA_C9, PA_C10, PA_C11, PA_C12, PA_C13, PA_CINTX, PA_CINTY, PA_NCOM };
enum : int {
  PA_MULTS = 4,         // pi8, pi10, pi11, pi13
  PA_EQS = 2,           // pix, piy
  PA_STEPS = 6,
  PA_DRAWS = 24,        // verifier draws: 5 per MultProof, 2 per EqualityProof
  PA_ENT_MULT0 = 4,     // MSM entries of a PointAddProof: C8 C10 C11 C13, then 6 per MultProof, then 2 per EqualityProof
  PA_ENT_EQ0 = 4 + 6 * PA_MULTS,
  PA_ENTRIES = PA_ENT_EQ0 + 2 * PA_EQS,
};
// statement (Cx, Cy, Cz) of MultProof m (pointAdd.ts:145-156)
ZK_LAYOUT_FN int pa_mult_com(int m, int k) {
  return m == 0 ? (k == 0 ? PA_C7 : k == 1 ? PA_C8 : PA_G)
       : m == 1 ? (k == 0 ? PA_C8 : k == 1 ? PA_C9 : PA_C10)
       : m == 2 ? (k == 0 ? PA_C10 : k == 1 ? PA_C10 : PA_C11)
       :          (k == 0 ? PA_C10 : k == 1 ? PA_C12 : PA_C13);
}
// statement (C1, C2) of EqualityProof e (pointAdd.ts:151-160)
ZK_LAYOUT_FN int pa_eq_com(int e, int k) { return e == 0 ? (k == 0 ? PA_C11 : PA_CINTX) : (k == 0 ? PA_C13 : PA_CINTY); }
// Challenges are indexed h = m for MultProof m and h = PA_MULTS + e for EqualityProof e.  The verifier aggregates
// (and draws) in the order pi8, pi10, pi11, pix, pi13, piy (pointAdd.ts:221-253): step s folds sub-proof pa_step(s)
// with the draws from pa_step_draw(s) on.
ZK_LAYOUT_FN int pa_step(int s) { return s == 3 ? PA_MULTS : s == 4 ? 3 : s; }
ZK_LAYOUT_FN int pa_step_draw(int s) { return s < 4 ? 5 * s : s == 4 ? 17 : 22; }   // 0 5 10 15 17 22
// index of a proof point (C8 C10 C11 C13 lead the PointAddProof) and of a derived point (DER_*), or -1
ZK_LAYOUT_FN int pa_point(int k) { return k == PA_C8 ? 0 : k == PA_C10 ? 1 : k == PA_C11 ? 2 : k == PA_C13 ? 3 : -1; }
ZK_LAYOUT_FN int pa_point_com(int i) { return i == 0 ? PA_C8 : i == 1 ? PA_C10 : i == 2 ? PA_C11 : PA_C13; }
ZK_LAYOUT_FN int pa_der(int k) {
  return k == PA_C7 ? DER_C7 : k == PA_C9 ? DER_C9 : k == PA_C12 ? DER_C12 : k == PA_CINTX ? DER_CINTX : k == PA_CINTY ? DER_CINTY : -1;
}
// byte offsets inside a PointAddProof
ZK_LAYOUT_FN int pa_mult_off(int m) { return 4 * WP + m * MULT_LEN; }
ZK_LAYOUT_FN int pa_eq_off(int e) { return 4 * WP + 4 * MULT_LEN + e * EQ_LEN; }
// encoding of commitment k: der = the five derived points (BSTRIDE apart, DER_* order), g = ProofGroup.g,
// pts = the four proof points (`stride` apart)
ZK_HD const uint8_t* pa_com_bytes(int k, const uint8_t* der, const uint8_t* g, const uint8_t* pts, size_t stride) {
  if (k == PA_G) return g;
  return pa_der(k) >= 0 ? der + (size_t)pa_der(k) * BSTRIDE : pts + (size_t)pa_point(k) * stride;
}

// Fiat-Shamir challenge of one sub-proof (mult.ts:116,156, equality.ts:69,101): H(statement, the proof's npts
// leading points).  s2 = null for an EqualityProof.
ZK_HD void sigma_challenge(uint32_t* c3, const uint8_t* s0, const uint8_t* s1, const uint8_t* s2, const uint8_t* pts, int npts) {
  Sha256 s;
  s.init();
  s.update(s0, WP);
  s.update(s1, WP);
  if (s2) s.update(s2, WP);
  s.update(pts, npts * WP);
  s.final80(c3);
}
// challenge h of the PointAddProof at pa (its points contiguous, the verifier's view): one hash state for both kinds of
// sub-proof, finalised once (VItemHashTask runs one thread per (sample, h))
ZK_HD void pa_challenge(uint32_t* c3, int h, const uint8_t* der, const uint8_t* g, const uint8_t* pa) {
  Sha256 s;
  s.init();
  if (h < PA_MULTS) {
    for (int k = 0; k < 3; k++) s.update(pa_com_bytes(pa_mult_com(h, k), der, g, pa, WP), WP);
    s.update(pa + pa_mult_off(h), 6 * WP);
  } else {
    for (int k = 0; k < 2; k++) s.update(pa_com_bytes(pa_eq_com(h - PA_MULTS, k), der, g, pa, WP), WP);
    s.update(pa + pa_eq_off(h - PA_MULTS), 2 * WP);
  }
  s.final80(c3);
}

// ---- derived commitments ------------------------------------------------------------------------------------------
// C7 = C2 - C1, C9 = C5 - C4, C12 = C1 - C3, Cint = C3 + C1 + C2, Cint2 = C4 + C6 (pointAdd.ts:137-159), each handed
// to out(DER_*, point) as soon as it is known.
template <class Out>
ZK_HD void point_add_derived(const Out& out, const TomPt& c1, const TomPt& c2, const TomPt& c3, const TomPt& c4,
                             const TomPt& c5, const TomPt& c6) {
  TomPt n, r;
  tom_neg(n, c1); tom_add(r, c2, n); out(DER_C7, r);
  tom_neg(n, c4); tom_add(r, c5, n); out(DER_C9, r);
  tom_neg(n, c3); tom_add(r, c1, n); out(DER_C12, r);
  tom_add(r, c3, c1); tom_add(r, r, c2); out(DER_CINTX, r);
  tom_add(r, c4, c6); out(DER_CINTY, r);
}
struct DerivedProj {   // stores the derived points projectively: point d at proj[first + d]
  uint32_t* proj;
  size_t first;         // (the sum is formed at each store: one 64-bit pointer fewer held across the additions)
  ZK_HD void operator()(int d, const TomPt& p) const { tom_st_xyz(proj + (first + d) * TOM_PROJ_WORDS, p.x, p.y, p.z); }
};
// coefficients of the statement C1..C6 once a coefficient of each derived commitment (a, indexed PA_*) is spread onto
// the points it is a sum of
ZK_HD void point_add_expand(uint32_t (*in)[8], const uint32_t (*a)[8]) {
  using F = Tomq;
  F::sub(in[0], a[PA_C12], a[PA_C7]); F::add(in[0], in[0], a[PA_CINTX]);   // C1: -C7 + C12 + Cint
  F::add(in[1], a[PA_C7], a[PA_CINTX]);                                   // C2:  C7 + Cint
  F::sub(in[2], a[PA_CINTX], a[PA_C12]);                                  // C3: -C12 + Cint
  F::sub(in[3], a[PA_CINTY], a[PA_C9]);                                   // C4: -C9 + Cint2
  copy_n<8>(in[4], a[PA_C9]);                                             // C5:  C9
  copy_n<8>(in[5], a[PA_CINTY]);                                          // C6:  Cint2
}

// ---- prover steps (mult.ts:93-131, equality.ts:60-78) --------------------------------------------------------------
// Every point a sub-proof emits is a commitment whose opening the prover knows, so the openings are handed to
// job(k, v, r) (canonical value and blinder of point k) for the fixed-base commitment kernel.  draw(q, r) yields the
// sub-proof's draw q, canonical.  All mod q = tom.order.
//
// MultProof with statement x, y (Montgomery) and blinder ry of Cy (Montgomery): points C4 Ax Ay Az A4_1 A4_2, draws
// k_x k_y k_z Ax.r Ay.r Az.r A4_1.r.  C4 = Cy*x = (x y) g + (x ry) h and A4_2 = Cy*k_x = (k_x y) g + (k_x ry) h
// (mult.ts:103-114).  Leaves r4 = x ry (Montgomery), the secret of t_r4.
template <class Job, class Draw>
ZK_HD void mult_openings(const Job& job, const Draw& draw, const uint32_t* xm, const uint32_t* ym, const uint32_t* rym,
                         uint32_t* r4) {
  using F = Tomq;
  uint32_t kx[8], ky[8], kz[8], mkx[8], ra[8], t[8], u[8];
  draw(0, kx);
  draw(1, ky);
  draw(2, kz);
  F::to_mont(mkx, kx);
  F::mul(t, xm, ym); F::from_mont(t, t);
  F::mul(r4, xm, rym); F::from_mont(u, r4);
  job(0, t, u);
  draw(3, ra); job(1, kx, ra);   // Ax, Ay, Az, A4_1 = commit(k_x), commit(k_y), commit(k_z), commit(k_z)
  draw(4, ra); job(2, ky, ra);
  draw(5, ra); job(3, kz, ra);
  draw(6, ra); job(4, kz, ra);
  F::mul(t, mkx, ym); F::from_mont(t, t);
  F::mul(u, mkx, rym); F::from_mont(u, u);
  job(5, t, u);
}
// EqualityProof: points A1 A2 = commit(k) under the blinders of draws 1 and 2, draws k A1.r A2.r
template <class Job, class Draw>
ZK_HD void equality_openings(const Job& job, const Draw& draw) {
  uint32_t k[8], ra[8];
  draw(0, k);
  draw(1, ra); job(0, k, ra);
  draw(2, ra); job(1, k, ra);
}
// response t = k - c*w  (mod q): k canonical, w Montgomery, c canonical 80-bit
ZK_HD void response(uint32_t* t, const uint32_t* k_canon, const uint32_t* cc, const uint32_t* w_mont) {
  using F = Tomq;
  uint32_t cw[8];
  F::mul(cw, cc, w_mont);   // c * (w R) / R = c*w, canonical
  F::sub(t, k_canon, cw);
}
// the NQ responses of a sub-proof (7 for a MultProof: t_x t_y t_z t_rx t_ry t_rz t_r4; 3 for an EqualityProof: t_x t_r1
// t_r2) to o: response q takes draw d0 + q of the tape row and the secret w(q, wm) (Montgomery).  cc: the challenge.
template <int NQ, class W>
ZK_HD void sigma_responses(ByteWriter& o, const uint32_t* cc, const uint8_t* row, int d0, const W& w) {
#pragma unroll
  for (int q = 0; q < NQ; q++) {
    uint32_t k[8], wm[8], t[8];
    tape_draw(k, row, d0 + q);
    reduce_once<FpP256>(k);
    w(q, wm);
    response(t, k, cc, wm);
    o.put_scalar<WS>(t);
  }
}

// ---- deserialisation checks (deserializePoint / deserializeScalar would throw) --------------------------------------
// Every check runs, so the thread does the same work on a valid and an invalid body.
ZK_HD bool valid_points(const uint8_t* p, int k) {
  bool ok = true;
  uint32_t x[PGL], y[PGL];
  for (int i = 0; i < k; i++) ok = tom_parse(x, y, p + (size_t)i * WP) && ok;
  return ok;
}
ZK_HD bool valid_scalars(const uint8_t* p, int k) {
  bool ok = true;
  uint32_t r[8];
  for (int i = 0; i < k; i++) ok = wscalar_parse(r, p + (size_t)i * WS) && ok;
  return ok;
}
ZK_HD bool valid_equality(const uint8_t* ep) { const bool ok = valid_points(ep, 2); return valid_scalars(ep + 2 * WP, 3) && ok; }
ZK_HD bool valid_mult(const uint8_t* mp) { const bool ok = valid_points(mp, 6); return valid_scalars(mp + 6 * WP, 7) && ok; }
ZK_HD bool valid_point_add(const uint8_t* pa) {
  bool ok = valid_points(pa, 4);
  for (int m = 0; m < PA_MULTS; m++) ok = valid_mult(pa + pa_mult_off(m)) && ok;
  for (int e = 0; e < PA_EQS; e++) ok = valid_equality(pa + pa_eq_off(e)) && ok;
  return ok;
}
// GK block of n rounds: n, then 4n points, then 3n + 1 scalars (gk.ts:208-218)
ZK_HD bool valid_gk(const uint8_t* g, int n) {
  const bool ok = valid_points(g + 1, 4 * n);
  return valid_scalars(g + 1 + (size_t)4 * n * WP, 3 * n + 1) && ok;
}

// ---- relation folds ------------------------------------------------------------------------------------------------
// The verifier's relations are linear combinations under fresh randomizers (Relation.drain).  A fold adds each term on
// a fixed base into gW / hW, each term on a statement commitment into that commitment's coefficient, and returns the
// scalars of the proof's own points.  All mod q = tom.order, Montgomery form unless said otherwise.
struct SigmaFold {
  uint32_t gW[8], hW[8];
  bool tape_ok;   // every draw was in range
};
struct Entries {  // MSM entries: canonical scalar and byte offset of the point
  uint32_t* scalar;
  uint32_t* off;
  ZK_HD void put(size_t i, const uint32_t* canon, uint32_t o) const {
    st<8>(scalar + i * 8, canon);
    off[i] = o;
  }
  ZK_HD void put_m(size_t i, const uint32_t* mont, uint32_t o) const {
    uint32_t v[8];
    Tomq::from_mont(v, mont);
    put(i, v, o);
  }
};
ZK_HD void challenge_mont(uint32_t* cm, const uint32_t* c3) {
  uint32_t cc[8];
  challenge_to_limbs(cc, c3);
  Tomq::to_mont(cm, cc);
}
// aggregateMult (mult.ts:148-175).  c3: challenge; mp: MultProof bytes; dr: its 5 draws; cx/cy/cz: coefficients of
// Cx, Cy, Cz; es: canonical scalars of C4 Ax Ay Az A4_1 A4_2.
ZK_HD void fold_mult(SigmaFold& f, const uint32_t* c3, const uint8_t* mp, const uint8_t* dr, uint32_t* cx, uint32_t* cy,
                     uint32_t* cz, uint32_t (*es)[8]) {
  using F = Tomq;
  uint32_t cm[8], ts[7][8], rr[5][8], rho[8], t0[8], coef[8], neg[8], z[8];
  challenge_mont(cm, c3);
  zero_n<8>(z);
  for (int q = 0; q < 7; q++) { wscalar_parse(ts[q], mp + 6 * WP + q * WS); F::to_mont(ts[q], ts[q]); }
  // ts: t_x t_y t_z t_rx t_ry t_rz t_r4
  for (int q = 0; q < 5; q++) { f.tape_ok = vdraw(rho, dr + 32 * q, false) && f.tape_ok; F::to_mont(rr[q], rho); }
  // rho1: t_x g + t_rx h + c Cx - A_x
  F::mul(t0, rr[0], ts[0]); F::add(f.gW, f.gW, t0);
  F::mul(t0, rr[0], ts[3]); F::add(f.hW, f.hW, t0);
  F::mul(coef, rr[0], cm); F::add(cx, cx, coef);
  F::sub(neg, z, rr[0]); F::from_mont(es[1], neg);
  // rho2: t_y g + t_ry h + c Cy - A_y ; rho5: t_x Cy + c C_4 - A_4_2
  F::mul(t0, rr[1], ts[1]); F::add(f.gW, f.gW, t0);
  F::mul(t0, rr[1], ts[4]); F::add(f.hW, f.hW, t0);
  F::mul(coef, rr[1], cm);
  F::mul(t0, rr[4], ts[0]); F::add(coef, coef, t0);
  F::add(cy, cy, coef);
  F::sub(neg, z, rr[1]); F::from_mont(es[2], neg);
  // rho3: t_z g + t_rz h + c Cz - A_z
  F::mul(t0, rr[2], ts[2]); F::add(f.gW, f.gW, t0);
  F::mul(t0, rr[2], ts[5]); F::add(f.hW, f.hW, t0);
  F::mul(coef, rr[2], cm); F::add(cz, cz, coef);
  F::sub(neg, z, rr[2]); F::from_mont(es[3], neg);
  // rho4: t_z g + t_r4 h + c C_4 - A_4_1
  F::mul(t0, rr[3], ts[2]); F::add(f.gW, f.gW, t0);
  F::mul(t0, rr[3], ts[6]); F::add(f.hW, f.hW, t0);
  F::add(coef, rr[3], rr[4]); F::mul(coef, coef, cm); F::from_mont(es[0], coef);   // C_4: (rho4 + rho5) c
  F::sub(neg, z, rr[3]); F::from_mont(es[4], neg);
  F::sub(neg, z, rr[4]); F::from_mont(es[5], neg);
}
// aggregateEquality (equality.ts:94-116).  ep: EqualityProof bytes; dr: its 2 draws; c1/c2: coefficients of C1, C2;
// es: canonical scalars of A1, A2.
ZK_HD void fold_equality(SigmaFold& f, const uint32_t* c3, const uint8_t* ep, const uint8_t* dr, uint32_t* c1, uint32_t* c2,
                         uint32_t (*es)[8]) {
  using F = Tomq;
  uint32_t cm[8], tx[8], tr1[8], tr2[8], ra[8], rb[8], rho[8], t0[8], t1[8], coef[8], neg[8], z[8];
  challenge_mont(cm, c3);
  zero_n<8>(z);
  wscalar_parse(tx, ep + 2 * WP); F::to_mont(tx, tx);
  wscalar_parse(tr1, ep + 2 * WP + WS); F::to_mont(tr1, tr1);
  wscalar_parse(tr2, ep + 2 * WP + 2 * WS); F::to_mont(tr2, tr2);
  f.tape_ok = vdraw(rho, dr, false) && f.tape_ok; F::to_mont(ra, rho);
  f.tape_ok = vdraw(rho, dr + 32, false) && f.tape_ok; F::to_mont(rb, rho);
  F::add(t1, ra, rb); F::mul(t0, t1, tx); F::add(f.gW, f.gW, t0);
  F::mul(t0, ra, tr1); F::add(f.hW, f.hW, t0);
  F::mul(t0, rb, tr2); F::add(f.hW, f.hW, t0);
  F::mul(coef, ra, cm); F::add(c1, c1, coef);
  F::mul(coef, rb, cm); F::add(c2, c2, coef);
  F::sub(neg, z, ra); F::from_mont(es[0], neg);
  F::sub(neg, z, rb); F::from_mont(es[1], neg);
}
// aggregatePointAdd (pointAdd.ts:199-259) of the PointAddProof at pa, whose byte offset in the caller's row is off.
// chal: the six challenges (3 words each, indexed h); dr: the PA_DRAWS draws.  Leaves in a[] one coefficient per
// commitment (g already folded into gW) and writes the PA_ENTRIES entries of its own points from `base` on.
ZK_HD void fold_point_add(SigmaFold& f, uint32_t (*a)[8], const uint32_t* chal, const uint8_t* pa, const uint8_t* dr,
                          const Entries& out, size_t base, uint32_t off) {
#pragma unroll
  for (int k = 0; k < PA_NCOM; k++) zero_n<8>(a[k]);
  uint32_t es[6][8];
#pragma unroll
  for (int s = 0; s < PA_STEPS; s++) {   // unrolled: the indices into a[] are compile-time
    const int h = pa_step(s);
    const uint8_t* ds = dr + 32 * pa_step_draw(s);
    if (h < PA_MULTS) {
      fold_mult(f, chal + 3 * h, pa + pa_mult_off(h), ds, a[pa_mult_com(h, 0)], a[pa_mult_com(h, 1)], a[pa_mult_com(h, 2)], es);
#pragma unroll
      for (int i = 0; i < 6; i++) out.put(base + PA_ENT_MULT0 + 6 * h + i, es[i], off + pa_mult_off(h) + i * WP);
    } else {
      const int e = h - PA_MULTS;
      fold_equality(f, chal + 3 * h, pa + pa_eq_off(e), ds, a[pa_eq_com(e, 0)], a[pa_eq_com(e, 1)], es);
#pragma unroll
      for (int i = 0; i < 2; i++) out.put(base + PA_ENT_EQ0 + 2 * e + i, es[i], off + pa_eq_off(e) + i * WP);
    }
  }
#pragma unroll
  for (int i = 0; i < 4; i++) out.put_m(base + i, a[pa_point_com(i)], off + i * WP);
  Tomq::add(f.gW, f.gW, a[PA_G]);   // C_14 = g
}

}  // namespace zk
