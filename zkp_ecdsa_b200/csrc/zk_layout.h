// zk_layout.h — byte layout of the flat proof and index maps shared by kernels and host.
//
// The flat layout is the concatenation of the reference's own primitives in class-field
// order (see include/zkattest.h and oracle/flat.py for the grammar):
//   Point.toBytes(): /root/reference/src/curves/weier.ts:244-255 (65 B),
//                    /root/reference/src/curves/edwards.ts:195-203 (67 B)
//   Scalar.toBytes(): /root/reference/src/curves/group.ts:196-199 (32 B p256 / 33 B tom)
#pragma once
#include <stdint.h>

#include "zkattest.h"  // status codes (one per reference throw site)

#if defined(__CUDACC__)
#define ZK_LAYOUT_FN __host__ __device__ inline constexpr
#else
#define ZK_LAYOUT_FN inline constexpr
#endif

namespace zk {

enum : int {
  NP = 65,   // P-256 point bytes
  NS = 32,   // P-256 scalar bytes
#if defined(ZKA_PG_WAR256)
  // ProofGroup = war256 (instances.ts:34-41): SEC1 points like P-256, scalars sized by its 256-bit field
  WP = 65,
  WS = 32,
  WCB = 32,  // bytes of one coordinate
#else
  WP = 67,   // tomEdwards256 point bytes
  WS = 33,   // tomEdwards256 scalar bytes (sized by the 258-bit FIELD, group.ts:49-52)
  WCB = 33,
#endif
  EQ_LEN = 2 * WP + 3 * WS,                       // 233 (tomEdwards256 sizes)  EqualityProof (equality.ts:28-32)
  MULT_LEN = 6 * WP + 7 * WS,                     // 633  MultProof     (mult.ts:27-39)
  PA_LEN = 4 * WP + 4 * MULT_LEN + 2 * EQ_LEN,    // 3266 PointAddProof (pointAdd.ts:29-38)
  REP_HEAD = 1 + NP + 2 * WP,                     // tag A Tx Ty
  REP1_LEN = REP_HEAD + 2 * NS + 2 * WS,          // 330  (exp.ts:31-34)
  REP0_LEN = REP_HEAD + 2 * NS + PA_LEN + 2 * WS, // 3596 (exp.ts:36-40)
  HEAD_LEN = 2 * NP + 2 * WP,                     // 264  R comS1 keyXcom keyYcom
  MAX_REPS = 80,
  // stride of one encoded point (65 or 67 bytes) in the byte stores: a multiple of 16, so that every staged encoding
  // starts on a 16-byte boundary and moves in five 16-byte transactions (a staging layout, not part of the proof format)
  BSTRIDE = 80,
};

ZK_LAYOUT_FN int gk_len(int n) { return 1 + 4 * n * WP + (3 * n + 1) * WS; }
ZK_LAYOUT_FN int proof_len(int zero_bits, int n, int reps) {
  return HEAD_LEN + zero_bits * REP0_LEN + (reps - zero_bits) * REP1_LEN + gk_len(n);
}

// ---- randomness tape: index of each 32-byte draw (SURVEY.md 3.1; reference call order) ----
enum : int {
  DRAW_COMS1_R = 0,   // pedersen.ts:54 via zkpAttestList.ts:138   (mod p256.n)
  DRAW_PKX_R = 1,     // zkpAttestList.ts:139                      (mod tom.order)
  DRAW_PKY_R = 2,     // zkpAttestList.ts:140
  DRAW_REP0 = 3,      // exp.ts:145-155: alpha_i, r_i (mod n), Tx_i.r, Ty_i.r (mod order)
  DRAWS_PER_REP = 4,
  DRAWS_PER_ITEM = 40,  // one 0-bit repetition: exp.ts:200-201 + pointAdd.ts:137-160
  // offsets inside an item
  IT_T1X_R = 0, IT_T1Y_R = 1, IT_C8_R = 2, IT_C10_R = 3, IT_C11_R = 4, IT_C13_R = 5,
  IT_MULT0 = 6,   // 4 MultProofs x [k_x,k_y,k_z,Ax.r,Ay.r,Az.r,A4_1.r] at 6,13,20 and 30
  IT_EQ0 = 27,    // pi_x [k, A1.r, A2.r]
  IT_MULT3 = 30,
  IT_EQ1 = 37,    // pi_y
  DRAWS_PER_GK_ROUND = 5,  // gk.ts:117-123: ri, ai, si, ti, rho_i
};
ZK_LAYOUT_FN int draws_before_items(int reps) { return DRAW_REP0 + DRAWS_PER_REP * reps; }
ZK_LAYOUT_FN int prove_draws(int zero_bits, int n, int reps) {
  return draws_before_items(reps) + DRAWS_PER_ITEM * zero_bits + DRAWS_PER_GK_ROUND * n;
}
ZK_LAYOUT_FN int item_mult_draw(int m) { return m < 3 ? IT_MULT0 + 7 * m : IT_MULT3; }

// ---- tomEdwards256 commitment jobs of one 0-bit repetition (34) and derived points (5) ----
enum : int {
  JOB_T1X = 0, JOB_T1Y = 1, JOB_C8 = 2, JOB_C10 = 3, JOB_C11 = 4, JOB_C13 = 5,
  JOB_MULT0 = 6,   // + 6*m + {C4, Ax, Ay, Az, A4_1, A4_2}
  JOB_EQ0 = 30,    // + 2*e + {A1, A2}
  JOBS_PER_ITEM = 34,
  DER_C7 = 0, DER_C9 = 1, DER_C12 = 2, DER_CINTX = 3, DER_CINTY = 4,
  DERS_PER_ITEM = 5,
  HASHES_PER_ITEM = 6,   // pi8, pi10, pi11, pi13, pix, piy (challenge order index)
  SECRETS_PER_ITEM = 34, // 4 x (x,y,z,rx,ry,rz,r4) + 2 x (x,r1,r2), Montgomery mod tom.order
};

}  // namespace zk
