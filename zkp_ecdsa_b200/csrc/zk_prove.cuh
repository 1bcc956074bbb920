// zk_prove.cuh — stage tasks of the batched prover (proveSignatureList over B proofs).
//
// Reference call tree being replaced (per proof):
//   /root/reference/src/zkpAttestList.ts:104-145  proveSignatureList
//   /root/reference/src/exp/exp.ts:126-231        proveExp        (80 cut-and-choose reps)
//   /root/reference/src/exp/pointAdd.ts:92-163    provePointAdd   (per 0-bit rep)
//   /root/reference/src/commit/mult.ts:93-131     proveMult       (4 per pointAdd)
//   /root/reference/src/commit/equality.ts:60-78  proveEquality   (2 per pointAdd)
//   /root/reference/src/proofGK/gk.ts:94-195      proveMembership
//
// Key restructuring (results identical, only affine encodings are observable):
//  * every tomEdwards256 point the prover emits is a commitment whose opening (v, r) the
//    prover knows — including the reference's variable-base products C4 = Cy*x and
//    A4_2 = Cy*k_x (mult.ts:103,114), since Cy = y*g + ry*h gives Cy*x = (xy)*g + (x ry)*h.
//    All ~1 560 Tom scalar multiplications per proof therefore run on the two fixed-base
//    tables of g and h (TomCommitTask) with scalars computed mod tom.order = p256.p.
//  * derived commitments C7, C9, C12, Cint (pointAdd.ts:137-159) are single point additions.
//  * all commitments of all repetitions of all proofs of a stage form ONE batch; the
//    Fiat-Shamir hashes are the only sequencing points.
#pragma once
#include "zk_sigma.cuh"

namespace zk {

struct ProveCtx {
  // dimensions
  int B;        // proofs in this chunk
  int S;        // repetitions (SecLevel, <= 80)
  int N;        // ring size
  int n;        // the depth the chunk is laid out for (grids, workspace strides, slots per proof): ceil(log2 N), with a
                //    ring set the largest depth the call uses; the depth of row b's own ring is n_row(b)
  int M;        // total 0-bit repetitions (items) in the chunk (valid after the scan)
  FbShape tom;                 // shape of the proof group's two fixed-base tables (g, h)
  int mode;                  // 0: proveSignatureList; 1: proveExp alone (exp.ts:126-231): R = `base`, s and Q are inputs,
                             //    the row holds the repetitions only (no header, no GK block)
  int head_len;              // bytes before the first repetition (HEAD_LEN, or 0 in mode 1)
  const uint8_t* base;       // mode 1: [B][65] paramsNIST.g
  const uint8_t* s_in;       // mode 1: [B][32] the committed exponent
  const uint8_t* q_in;       // mode 1: [B][65] Q (65 zero bytes = identity) or null
  uint32_t* base_aff;        // [B][16] base of the per-key tables: pk in mode 0, `base` in mode 1
  // inputs (device copies)
  const uint8_t* msg_hash;   // [B][32]
  const uint8_t* sig;        // [B][64]
  const uint8_t* pk;         // [B][65]
  const uint32_t* which;     // [B]  caller's index (only range-checked: RPointTask)
  uint32_t* which_s;         // [B]  sanitised copy (0 when outside the ring): every ring_m / bit access uses this one
  const uint8_t* tape;       // [B][tape_stride]
  size_t tape_stride;
  uint32_t tape_draws;       // draws available per proof
  const uint32_t* ring_m;    // [2^n] ring values mod tom.order, Montgomery, padded with ring[0]; with a ring set, every
                             //    ring of the set (zka_rings), ring r at entry ring_base[r]
  const uint32_t* ring_of;   // [B] ring-set calls: the ring of each row (null: every row uses ring_m, N entries)
  const uint32_t* ring_base; // [R] entry offset of each padded ring of the set
  const uint32_t* ring_size; // [R] N_r
  const uint32_t* ring_depth;// [R] n_r = ceil(log2 N_r) <= n
  // parameters / tables
  const uint32_t* g_tab8;    // P-256 generator, w=8 affine table [32][256][16]
  const uint32_t* h_tab8;    // NistGroup.h, fixed-base affine table with h_w-bit windows
  int h_w;
  const uint32_t* g_tabw;    // P-256 generator again, with g_w-bit windows (phase A)
  int g_w;
  const uint32_t* tg_tab;    // ProofGroup.g table [nwin][2^w][32]
  const uint32_t* th_tab;    // ProofGroup.h table
  const uint8_t* tg_bytes;   // 67-byte encoding of ProofGroup.g (C_14, pointAdd.ts:144)
  // per proof state
  uint32_t* s1;        // [B][8]  s1 canonical mod n
  uint32_t* pk_aff;    // [B][16] pk affine Montgomery
  uint32_t* q_aff;     // [B][16] Q = z1*G
  uint8_t* q_inf;      // [B]
  uint32_t* r_aff;     // [B][16] R
  uint8_t* r_bytes;    // [B][BSTRIDE]
  uint32_t* u12;       // [B][16] u1 = z/s, u2 = r/s (Montgomery mod n): R = u1*G + u2*pk
  uint32_t* tab_of;    // [B]   table index of the proof's pk (equal keys of a batch share one table)
  uint32_t* tab_rep;   // [B]   proof index that owns table t; tab_count[0] = number of tables
  uint32_t* tab_count; // [2]   [0] number of tables, [1] their window bits (key_window_bits)
  uint32_t* rpows;     // [B][52][24]               per-KEY signed-digit table of pk (window bits tab_count[1]):
  uint32_t* rrows;     // [B * KEY_CAP][24]           every alpha*R of the proof is evaluated as
  uint32_t* rtab;      // [B * KEY_CAP][16]           (alpha u1)*G + (alpha u2)*pk, so no table of R is needed
  // phase A (P-256): slot i in [0,S] per proof; slot S is comS1
  uint32_t* pa_T;      // [B][S+1][24]
  uint32_t* pa_A;      // [B][S+1][24]
  uint32_t* pa_T_aff;  // [B][S+1][16]
  uint8_t* pa_T_inf;   // [B][S+1]
  uint32_t* pa_A_aff;  // [B][S+1][16] (unused values, bytes matter)
  uint8_t* pa_A_bytes; // [B][S+1][BSTRIDE]
  uint8_t* pa_A_inf;   // [B][S+1]
  // Tom store 1 (pre-challenge): per proof 2 + 2S points: pkX, pkY, (Tx_i, Ty_i)
  uint32_t *s1_jv, *s1_jr, *s1_proj, *s1_aff;
  uint8_t* s1_bytes;
  // challenge / items
  uint32_t* chal;      // [B][3]  80-bit exp challenge
  uint32_t* zcount;    // [B]     zero bits
  uint32_t* item_base; // [B]     exclusive prefix of zcount
  uint32_t* item_total;// [1]
  uint32_t* rep_off;   // [B][S]  byte offset of each repetition inside the proof
  uint32_t* gk_off;    // [B]     byte offset of the GK proof
  uint32_t* item_b;    // [M]     proof of item
  uint32_t* item_i;    // [M]     repetition of item
  uint32_t* item_k;    // [M]     rank of the item among the proof's zero bits
  // phase B (P-256)
  uint32_t* pb_T1;     // [M][24]
  uint32_t* pb_T1_aff; // [M][16]
  uint8_t* pb_T1_inf;  // [M]
  // Tom store 2 (post-challenge): [34 M jobs][5 M derived][4n B GK]
  uint32_t *s2_jv, *s2_jr, *s2_proj, *s2_aff;
  uint8_t* s2_bytes;
  uint32_t* item_inv;  // [M][8]     1 / (x2 - x1) of the item's point addition (Montgomery mod q; 0 for 0)
  uint32_t* secrets;   // [M][34][8] Montgomery mod tom.order
  uint32_t* item_chal; // [M][6][3]
  // GK
  uint32_t* gk_dv;     // [B][n][8]  d(omega_w), Montgomery (row b fills its first n_row(b))
  uint32_t* gk_part;   // [B][n][2^(n-k)][8] block sums of d(omega_w) when the ring is cut into blocks (n > k)
  uint32_t* gk_lag;    // [n][n][8]  Lagrange matrix for nodes 0..n-1, Montgomery; with a ring set the matrices of every
                       //    depth 1..n, depth d at word gk_lag_off(d)
  uint32_t* gk_x;      // [B][3]
  // outputs
  uint8_t* proofs;     // [B][proof_stride]
  size_t proof_stride;
  uint32_t* proof_len; // [B]
  int32_t* status;     // [B]

  ZK_HD size_t s2_job(size_t item, int j) const { return item * JOBS_PER_ITEM + j; }
  ZK_HD size_t s2_der(size_t item, int j) const { return (size_t)M * JOBS_PER_ITEM + item * DERS_PER_ITEM + j; }
  // GK commitment j of row b: cl ca cb cd fill the first 4 n_row(b) of the row's 4n slots, the rest are zero jobs
  ZK_HD size_t s2_gk(size_t b, int j) const { return (size_t)M * (JOBS_PER_ITEM + DERS_PER_ITEM) + b * 4 * n + j; }
  ZK_HD size_t s2_count() const { return (size_t)M * (JOBS_PER_ITEM + DERS_PER_ITEM) + (size_t)B * 4 * n; }
  ZK_HD size_t s1_pt(size_t b, int j) const { return b * (2 + 2 * S) + j; }  // 0 pkX, 1 pkY, 2+2i Tx_i, 3+2i Ty_i
  ZK_HD const uint8_t* tape_of(int b) const { return tape + (size_t)b * tape_stride; }
  // the ring of row b (its 2^n padded entries) and its size
  ZK_HD const uint32_t* ring_of_row(int b) const { return ring_of ? ring_m + (size_t)8 * ring_base[ring_of[b]] : ring_m; }
  ZK_HD uint32_t ring_size_row(int b) const { return ring_of ? ring_size[ring_of[b]] : (uint32_t)N; }
  // the depth of row b's ring, the n of its proof (gk.ts:94-195), and the Lagrange matrix of that depth
  ZK_HD int n_row(int b) const { return ring_of ? (int)ring_depth[ring_of[b]] : n; }
  ZK_HD static size_t gk_lag_off(int d) { return (size_t)8 * ((size_t)(d - 1) * d * (2 * d - 1) / 6); }   // 8 * sum of e^2, e < d
  ZK_HD const uint32_t* gk_lag_row(int b) const { return ring_of ? gk_lag + gk_lag_off(n_row(b)) : gk_lag; }
};

// draw a scalar and check it is below the modulus (the host pre-filters, see include/zkattest.h)
template <class F>
ZK_HD bool draw_checked(uint32_t* r, const ProveCtx& c, int b, int draw) {
  if ((uint32_t)draw >= c.tape_draws) {
    zero_n<8>(r);
    ZK_SET_STATUS(c.status + b, ZKA_ERR_TAPE_RANGE);
    return false;
  }
  tape_draw(r, c.tape_of(b), draw);
  if (!lt_p<F>(r)) {
    ZK_SET_STATUS(c.status + b, ZKA_ERR_TAPE_RANGE);
    sub_p<F>(r, r);  // keep arithmetic well defined; the proof is flagged anyway
    return false;
  }
  return true;
}

// ---------------------------------------------------------------------------------------------
// Stage 0 — ECDSA statement (zkpAttestList.ts:112-136): one thread per proof.
//   u1 = z/s, u2 = r/s, s1 = s/r, Q = z1*G  (invMod(0) = 0 as in big.ts).
// R = u1*G + u2*pk is NOT computed here with a variable-base ladder (a 256-doubling latency chain per
// proof).  The pipeline builds ONE positional table per proof, of pk, and evaluates R (RPointTask) and
// every alpha*R of phase A on the G table and that pk table.
// ---------------------------------------------------------------------------------------------
struct PreKeyTask {   // validate and store the public key (everything the key tables depend on)
  ProveCtx c;
  ZK_HD void operator()(int b) const {
    c.status[b] = ZKA_OK;
    P256Aff pk;
    bool inf;
    if (!p256_parse(pk, inf, c.pk + (size_t)b * 65) || inf) {   // the identity is no key either
      ZK_SET_STATUS(c.status + b, ZKA_ERR_INVALID_PK);
      // keep going with the generator so later stages stay well defined
      p256_set_generator(pk);
    }
    p256_st_aff(c.pk_aff + (size_t)b * 16, pk);
    if (c.mode == 1) {   // the tables are built for paramsNIST.g, an input of its own
      P256Aff g;
      if (!p256_parse(g, inf, c.base + (size_t)b * 65) || inf) {
        ZK_SET_STATUS(c.status + b, ZKA_ERR_INVALID_PK);
        p256_set_generator(g);
      }
      p256_st_aff(c.base_aff + (size_t)b * 16, g);
      c.which_s[b] = 0;
      return;
    }
    // an index outside the ring is flagged by RPointTask (ZKA_ERR_BAD_INDEX); the Groth-Kohlweiss tasks
    // must still stay inside ring_m[2^n], so they read this clamped copy
    const uint32_t w = c.which[b];
    c.which_s[b] = w < c.ring_size_row(b) ? w : 0u;
  }
};
struct PreTask {      // the scalars of the statement and Q = z1*G
  ProveCtx c;
  ZK_HD void operator()(int b) const {
    using Fp = P256p;
    using Fn = P256n;
    if (c.mode == 1) {   // alpha*R = 0*G + alpha*base; s and Q are given
      uint32_t s1[8], u[8];
      limbs_from_be<8>(s1, c.s_in + (size_t)b * 32, 32);
      reduce_once<FnP256>(s1);
      st<8>(c.s1 + (size_t)b * 8, s1);
      zero_n<8>(u);
      st<8>(c.u12 + (size_t)b * 16, u);
      Fn::set_one(u);
      st<8>(c.u12 + (size_t)b * 16 + 8, u);
      P256Aff Qa;
      bool qinf = true;   // no Q, the identity, or an invalid Q (flagged): no Q term
      if (c.q_in && !p256_parse(Qa, qinf, c.q_in + (size_t)b * 65)) { ZK_SET_STATUS(c.status + b, ZKA_ERR_INVALID_PK); qinf = true; }
      if (qinf) p256_set_generator(Qa);
      p256_st_aff(c.q_aff + (size_t)b * 16, Qa);
      c.q_inf[b] = qinf ? 1 : 0;
      return;
    }
    uint32_t z[8], r[8], s[8];
    limbs_from_be<8>(z, c.msg_hash + (size_t)b * 32, 32);   // truncateToN is the identity for 32 bytes
    limbs_from_be<8>(r, c.sig + (size_t)b * 64, 32);
    limbs_from_be<8>(s, c.sig + (size_t)b * 64 + 32, 32);
    reduce_once<FnP256>(z);
    reduce_once<FnP256>(r);
    reduce_once<FnP256>(s);
    uint32_t zm[8], rm[8], sm[8], sinv[8], rinv[8], t[8];
    Fn::to_mont(zm, z);
    Fn::to_mont(rm, r);
    Fn::to_mont(sm, s);
    Fn::inv(sinv, sm);
    Fn::inv(rinv, rm);
    uint32_t s1[8], z1[8];
    Fn::mul(t, sinv, zm); st<8>(c.u12 + (size_t)b * 16, t);
    Fn::mul(t, sinv, rm); st<8>(c.u12 + (size_t)b * 16 + 8, t);
    Fn::mul(t, rinv, sm); Fn::from_mont(s1, t);
    Fn::mul(t, rinv, zm); Fn::from_mont(z1, t);
    st<8>(c.s1 + (size_t)b * 8, s1);

    // Q = z1*G, affine (own inversion: once per proof)
    P256Pt Q;
    p256_set_identity(Q);
    p256_accum_fixed(Q, c.g_tab8, z1, 8);
    uint32_t zi[8];
    P256Aff Qa;
    bool qinf = p256_is_identity(Q);
    if (qinf) {
      p256_set_generator(Qa);
    } else {
      Fp::inv(zi, Q.z);
      Fp::mul(Qa.x, Q.x, zi);
      Fp::mul(Qa.y, Q.y, zi);
    }
    p256_st_aff(c.q_aff + (size_t)b * 16, Qa);
    c.q_inf[b] = qinf ? 1 : 0;
  }
};

// Stage 0a — equal public keys share one table.  A chunk of Bc proofs holds up to Bc distinct keys (at most N when
// every proof of a one-ring call is made by a ring member, up to Bc with a ring set); tables (a 255-doubling chain,
// 780 additions and 832 normalisations each) are built per distinct key.  Thread b looks for the first proof with the same
// (validated, Montgomery-form) key; KeyRankTask turns first occurrences into dense table indices.
struct KeyDedupTask {
  ProveCtx c;
  ZK_HD void operator()(int b) const {
    uint32_t mine[16];
    ld<16>(mine, c.base_aff + (size_t)b * 16);
    int rep = b;
    for (int o = 0; o < b; o++) {
      const uint32_t* q = c.base_aff + (size_t)o * 16;
      if (q[0] != mine[0]) continue;
      bool same = true;
      for (int i = 1; i < 16; i++) same = same && (q[i] == mine[i]);
      if (same) { rep = o; break; }
    }
    c.tab_of[b] = (uint32_t)rep;      // provisional: index of the first proof with this key
  }
};
struct KeyRankTask {
  ProveCtx c;
  ZK_HD void operator()(int b) const {
    const uint32_t rep = c.tab_of[b];
    // (tab_of is only rewritten by the follow-up KeyAssignTask, so every thread sees first occurrences)
    uint32_t rank = 0;
    for (uint32_t o = 0; o < rep; o++) rank += (c.tab_of[o] == o) ? 1u : 0u;
    c.tab_rep[c.B + b] = rank;        // scratch half of tab_rep: rank of this proof's table
    if (rep == (uint32_t)b) c.tab_rep[rank] = (uint32_t)b;
    if (b == c.B - 1) {
      uint32_t total = 0;
      for (uint32_t o = 0; o < (uint32_t)c.B; o++) total += (c.tab_of[o] == o) ? 1u : 0u;
      c.tab_count[0] = total;
      c.tab_count[1] = (uint32_t)key_window_bits(total, (uint32_t)c.B, (uint32_t)c.S + 2);
    }
  }
};
struct KeyAssignTask {
  ProveCtx c;
  ZK_HD void operator()(int b) const { c.tab_of[b] = c.tab_rep[c.B + b]; }
};

// The doubling chains of the (few) distinct keys and the per-proof scalar stage are both latency bound
// and independent of each other: one grid runs them side by side.
struct PowsAndPreTask {
  P256PowsTask pows;
  PreTask pre;
  int Bp;   // pows.nbase rounded up to a warp multiple
  ZK_HD void operator()(int t) const {
    if (t < Bp) {
      if (t < pows.nbase) pows(t);
    } else if (t - Bp < pre.c.B) {
      pre(t - Bp);
    }
  }
};

// Stage 0b — R = u1*G + u2*pk on the tables, affine + encoded; per-proof checks in the reference's order.
struct RPointTask {
  ProveCtx c;
  ZK_HD void operator()(int b) const {
    using Fp = P256p;
    using Fn = P256n;
    uint32_t m[8], u1[8], u2[8];
    ld<8>(m, c.u12 + (size_t)b * 16);     Fn::from_mont(u1, m);
    ld<8>(m, c.u12 + (size_t)b * 16 + 8); Fn::from_mont(u2, m);
    P256Jac acc;
    p256_set_identity_jac(acc);
    p256_accum_fixed_jac(acc, c.g_tabw, u1, c.g_w);
    const int kw = (int)c.tab_count[1];
    p256_accum_fixed_jac(acc, c.rtab + (size_t)c.tab_of[b] * key_table_words(kw), u2, kw);
    P256Pt R;
    p256_jac_to_hom(R, acc);
    uint32_t zi[8];
    P256Aff Ra;
    if (p256_is_identity(R)) {
      ZK_SET_STATUS_OVER(c.status + b, ZKA_ERR_T_INFINITY, ZKA_ERR_TAPE_RANGE);  // T_i = R*alpha is the identity (exp.ts:151)
      p256_set_generator(Ra);
    } else {
      Fp::inv(zi, R.z);
      Fp::mul(Ra.x, R.x, zi);
      Fp::mul(Ra.y, R.y, zi);
    }
    if (c.mode == 0) {
      uint32_t r[8];
      limbs_from_be<8>(r, c.sig + (size_t)b * 64, 32);
      reduce_once<FnP256>(r);
      if (is_zero_n<8>(r)) ZK_SET_STATUS_OVER(c.status + b, ZKA_ERR_POINTS_DONT_ADD, ZKA_ERR_TAPE_RANGE);  // rinv = 0: T1 + pk != T (pointAdd.ts:105)
    }
    p256_st_aff(c.r_aff + (size_t)b * 16, Ra);
    uint8_t* rb = c.r_bytes + (size_t)b * BSTRIDE;
    uint32_t cv[8];
    rb[0] = 0x04;
    Fp::from_mont(cv, Ra.x); limbs_to_be<8>(rb + 1, cv, 32);
    Fp::from_mont(cv, Ra.y); limbs_to_be<8>(rb + 33, cv, 32);
    if (c.mode == 0 && c.which[b] >= c.ring_size_row(b)) ZK_SET_STATUS_OVER(c.status + b, ZKA_ERR_BAD_INDEX, ZKA_ERR_TAPE_RANGE);
  }
};

// ---------------------------------------------------------------------------------------------
// Stage 1 — exp.ts:144-148: T_i = alpha_i*R, A_i = T_i + r_i*h; slot S: comS1 = s1*R + r*h
// (zkpAttestList.ts:137-138).  One thread per (proof, slot).
//   alpha*R = (alpha u1 mod n)*G + (alpha u2 mod n)*pk
// ---------------------------------------------------------------------------------------------
struct PhaseAP256Task {
  ProveCtx c;
  ZK_HD void operator()(int t) const {
    using Fn = P256n;
    const int S1 = c.S + 1;
    const int b = t / S1, i = t % S1;
    uint32_t alpha[8], r[8];
    if (i < c.S) {
      draw_checked<FnP256>(alpha, c, b, DRAW_REP0 + DRAWS_PER_REP * i);
      draw_checked<FnP256>(r, c, b, DRAW_REP0 + DRAWS_PER_REP * i + 1);
    } else {
      ld<8>(alpha, c.s1 + (size_t)b * 8);
      draw_checked<FnP256>(r, c, b, DRAW_COMS1_R);
    }
    uint32_t am[8], um[8], pm[8], a1[8], a2[8];
    Fn::to_mont(am, alpha);
    ld<8>(um, c.u12 + (size_t)b * 16);     Fn::mul(pm, am, um); Fn::from_mont(a1, pm);
    ld<8>(um, c.u12 + (size_t)b * 16 + 8); Fn::mul(pm, am, um); Fn::from_mont(a2, pm);
    // one Jacobian accumulator through G -> key -> h; only T and A are converted (jac_to_hom keeps Z = 0 for the
    // identity, so P256NormTask's infinity flags are unchanged)
    P256Jac acc;
    p256_set_identity_jac(acc);
    p256_accum_fixed_jac(acc, c.g_tabw, a1, c.g_w);
    const int kw = (int)c.tab_count[1];
    p256_accum_fixed_jac(acc, c.rtab + (size_t)c.tab_of[b] * key_table_words(kw), a2, kw);
    P256Pt T, A;
    p256_jac_to_hom(T, acc);
    p256_accum_fixed_jac(acc, c.h_tab8, r, c.h_w);
    p256_jac_to_hom(A, acc);
    p256_st_proj(c.pa_T + (size_t)t * P256_PROJ_WORDS, T);
    p256_st_proj(c.pa_A + (size_t)t * P256_PROJ_WORDS, A);
  }
};

// (TaskMinBlocks<PhaseAP256Task> = 5, i.e. <= 102 registers so that 81 x 1024 threads fit one wave, spills
//  and did not help — left at the default.)

// (A two-thread-per-commitment phase A + combine pass for batches under two waves was slower than this
//  kernel — the halves repeat the scalar preparation and the digit recoding — and was removed again.)
// R itself is only needed after phase A (its encoding goes into the proof header), and phase A works on
// the tables: both run in one grid.  RPointTask's errors precede phase A's tape-range error in the
// pipeline order, hence ZK_SET_STATUS_OVER there.
struct PhaseAAndRPointTask {
  PhaseAP256Task pa;
  RPointTask rp;
  int nA, nAp;   // phase-A threads, rounded up to a warp multiple
  ZK_HD void operator()(int t) const {
    if (t < nAp) {
      if (t < nA) pa(t);
    } else if (t - nAp < rp.c.B) {
      rp(t - nAp);
    }
  }
};

// Stage 2a — commitment jobs for pkX, pkY (zkpAttestList.ts:139-140) and Tx_i, Ty_i
// (exp.ts:154-155).  One thread per (proof, j), j in [0, 2+2S).
struct JobsATask {
  ProveCtx c;
  ZK_HD void operator()(int t) const {
    using Fp = P256p;
    const int per = 2 + 2 * c.S;
    const int b = t / per, j = t % per;
    uint32_t v[8], r[8], m[8];
    if (j < 2) {
      ld8v(m, c.pk_aff + (size_t)b * 16 + 8 * j);
      draw_checked<FpP256>(r, c, b, DRAW_PKX_R + j);
    } else {
      const int i = (j - 2) >> 1, xy = (j - 2) & 1;
      const size_t slot = (size_t)b * (c.S + 1) + i;
      if (c.pa_T_inf[slot]) ZK_SET_STATUS(c.status + b, ZKA_ERR_T_INFINITY);   // exp.ts:150-152
      if (c.pa_A_inf[slot]) ZK_SET_STATUS(c.status + b, ZKA_ERR_IDENTITY_ENC);
      ld8v(m, c.pa_T_aff + slot * 16 + 8 * xy);
      draw_checked<FpP256>(r, c, b, DRAW_REP0 + DRAWS_PER_REP * i + 2 + xy);
    }
    Fp::from_mont(v, m);  // coordinate as an integer: a scalar of the proof group
    st8v(c.s1_jv + (size_t)t * 8, v);
    st8v(c.s1_jr + (size_t)t * 8, r);
  }
};

// Stage 3 — exp.ts:158-165 challenge = H(pkX, pkY, A_0, Tx_0, Ty_0, ...); per proof.
// Also lays the proof out: repetition offsets, item ranks, header + tags.
struct ExpChallengeTask {
  ProveCtx c;
  struct Src {
    const ProveCtx* c;
    int b;
    ZK_HD const uint8_t* operator()(int k, int& len) const {
      if (k < 2) { len = WP; return c->s1_bytes + c->s1_pt(b, k) * BSTRIDE; }
      const int i = (k - 2) / 3, w = (k - 2) % 3;
      if (w == 0) { len = NP; return c->pa_A_bytes + ((size_t)b * (c->S + 1) + i) * BSTRIDE; }
      len = WP;
      return c->s1_bytes + c->s1_pt(b, 2 + 2 * i + (w - 1)) * BSTRIDE;
    }
  };
  ZK_HD void operator()(int b) const {
    uint32_t c3[3];
    Src src{&c, b};
    hash_points80(c3, src, 2 + 3 * c.S);
    st<3>(c.chal + (size_t)b * 3, c3);
    uint32_t off = (uint32_t)c.head_len, z = 0;
    for (int i = 0; i < c.S; i++) {
      const uint32_t bit = (c3[i >> 5] >> (i & 31)) & 1u;   // LSB first (exp.ts:169,228)
      c.rep_off[(size_t)b * c.S + i] = off;
      off += bit ? REP1_LEN : REP0_LEN;
      z += bit ? 0 : 1;
    }
    c.zcount[b] = z;
    c.gk_off[b] = off;
    c.proof_len[b] = c.mode == 1 ? off : off + gk_len(c.n_row(b));
  }
};
// single-thread exclusive scan of zcount (B <= a few thousand per chunk)
struct ScanTask {
  ProveCtx c;
  ZK_HD void operator()(int) const {
    uint32_t acc = 0, mx = 0;
    for (int b = 0; b < c.B; b++) {
      c.item_base[b] = acc;
      acc += c.zcount[b];
      if (c.zcount[b] > mx) mx = c.zcount[b];
    }
    c.item_total[0] = acc;
    c.item_total[1] = mx;   // longest proof of the chunk (bounds the D2H row width)
  }
};
struct ItemsTask {
  ProveCtx c;
  ZK_HD void operator()(int b) const {
    uint32_t c3[3];
    ld<3>(c3, c.chal + (size_t)b * 3);
    uint32_t k = 0;
    for (int i = 0; i < c.S; i++) {
      const uint32_t bit = (c3[i >> 5] >> (i & 31)) & 1u;
      if (!bit) {
        const uint32_t it = c.item_base[b] + k;
        c.item_b[it] = b;
        c.item_i[it] = i;
        c.item_k[it] = k;
        k++;
      }
    }
  }
};

// Stage 4 — exp.ts:186-190: z = alpha_i - s1, T1 = z*R + Q.  Because the statement was built as
// R = (z/s) G + (r/s) pk, s1 = s/r, Q = (z/r) G, the identity s1*R - Q = pk holds whenever r and s
// are invertible (otherwise PreTask has already flagged the proof), hence
//     T1 = alpha_i*R - (s1*R - Q) = T_i - pk :
// one complete mixed addition per item instead of a 64-lookup scalar multiplication.
struct PhaseBP256Task {
  ProveCtx c;
  ZK_HD void operator()(int it) const {
    using F = P256p;
    const int b = c.item_b[it], i = c.item_i[it];
    const size_t slot = (size_t)b * (c.S + 1) + i;
    P256Aff T, npk;
    p256_ld_aff(T, c.pa_T_aff + slot * 16);
    p256_ld_aff(npk, c.pk_aff + (size_t)b * 16);
    F::neg(npk.y, npk.y);
    P256Pt T1;
    if (c.pa_T_inf[slot]) p256_set_identity(T1); else p256_from_affine(T1, T);
    p256_madd(T1, T1, npk);
    p256_st_proj(c.pb_T1 + (size_t)it * P256_PROJ_WORDS, T1);
  }
};

// Stage 5a — the one inversion of every item, i8 = 1 / (x2 - x1) (pointAdd.ts:131), batched:
// one thread runs Montgomery's trick over ITEM_INV_CHUNK items (one binary inversion instead of 8).
// invMod(0) = 0 as in big.ts: a zero difference is replaced by 1 inside the product and yields 0.
enum : int { ITEM_INV_CHUNK = 8 };
struct ItemInvTask {
  ProveCtx c;
  ZK_HD void operator()(int t) const {
    using F = Tomq;
    const int lo = t * ITEM_INV_CHUNK;
    int n = c.M - lo;
    if (n > ITEM_INV_CHUNK) n = ITEM_INV_CHUNK;
    uint32_t d[ITEM_INV_CHUNK][8], pre[ITEM_INV_CHUNK][8], acc[8];
    bool z[ITEM_INV_CHUNK];
    F::set_one(acc);
#pragma unroll
    for (int k = 0; k < ITEM_INV_CHUNK; k++) {
      if (k < n) {
        const int it = lo + k;
        uint32_t x1[8], x2[8], one[8];
        ld<8>(x1, c.pb_T1_aff + (size_t)it * 16);
        ld<8>(x2, c.pk_aff + (size_t)c.item_b[it] * 16);
        F::sub(d[k], x2, x1);
        z[k] = is_zero_n<8>(d[k]);
        F::set_one(one);
        csel_n<8>(d[k], z[k], one, d[k]);
        F::mul(acc, acc, d[k]);
        copy_n<8>(pre[k], acc);
      }
    }
    uint32_t inv[8];
    F::inv(inv, acc);
#pragma unroll
    for (int k = ITEM_INV_CHUNK - 1; k >= 0; k--) {
      if (k < n) {
        uint32_t r[8], zero[8];
        if (k > 0) F::mul(r, inv, pre[k - 1]); else copy_n<8>(r, inv);
        F::mul(inv, inv, d[k]);
        zero_n<8>(zero);
        csel_n<8>(r, z[k], zero, r);
        st<8>(c.item_inv + (size_t)(lo + k) * 8, r);
      }
    }
  }
};

// ---------------------------------------------------------------------------------------------
// Stage 5 — pointAdd.ts:125-160 witnesses + every commitment opening of one 0-bit repetition,
// in the proof-group scalar field F_q, q = tom.order = p256.p.  One thread per item.
// ---------------------------------------------------------------------------------------------
struct ItemScalarsTask {
  ProveCtx c;
  ZK_HD void job(size_t item, int j, const uint32_t* v_mont, const uint32_t* r_canon) const {
    uint32_t v[8];
    Tomq::from_mont(v, v_mont);
    st8v(c.s2_jv + c.s2_job(item, j) * 8, v);
    st8v(c.s2_jr + c.s2_job(item, j) * 8, r_canon);
  }
  ZK_HD void job_raw(size_t item, int j, const uint32_t* v, const uint32_t* r) const {
    st8v(c.s2_jv + c.s2_job(item, j) * 8, v);
    st8v(c.s2_jr + c.s2_job(item, j) * 8, r);
  }
  ZK_HD void operator()(int it) const {
    using F = Tomq;
    const int b = c.item_b[it], i = c.item_i[it], k = c.item_k[it];
    if (c.pb_T1_inf[it]) ZK_SET_STATUS(c.status + b, ZKA_ERR_T1_INFINITY);  // exp.ts:192-194
    const int d0 = draws_before_items(c.S) + DRAWS_PER_ITEM * k;
    // coordinates (Montgomery residues mod p256.p double as F_q elements)
    uint32_t x1[8], y1[8], x2[8], y2[8], x3[8];
    ld8v(x1, c.pb_T1_aff + (size_t)it * 16);
    ld8v(y1, c.pb_T1_aff + (size_t)it * 16 + 8);
    ld8v(x2, c.pk_aff + (size_t)b * 16);
    ld8v(y2, c.pk_aff + (size_t)b * 16 + 8);
    ld8v(x3, c.pa_T_aff + ((size_t)b * (c.S + 1) + i) * 16);
    // blinders (canonical) and their Montgomery forms
    uint32_t rT1x[8], rT1y[8], rPkx[8], rPky[8], rTx[8], rTy[8];
    draw_checked<FpP256>(rT1x, c, b, d0 + IT_T1X_R);
    draw_checked<FpP256>(rT1y, c, b, d0 + IT_T1Y_R);
    draw_checked<FpP256>(rPkx, c, b, DRAW_PKX_R);
    draw_checked<FpP256>(rPky, c, b, DRAW_PKY_R);
    draw_checked<FpP256>(rTx, c, b, DRAW_REP0 + DRAWS_PER_REP * i + 2);
    draw_checked<FpP256>(rTy, c, b, DRAW_REP0 + DRAWS_PER_REP * i + 3);
    uint32_t mT1x[8], mT1y[8], mPkx[8], mPky[8], mTx[8], mTy[8];
    F::to_mont(mT1x, rT1x); F::to_mont(mT1y, rT1y);
    F::to_mont(mPkx, rPkx); F::to_mont(mPky, rPky);
    F::to_mont(mTx, rTx);   F::to_mont(mTy, rTy);
    // pointAdd.ts:130-136
    uint32_t i7[8], i8[8], i9[8], i10[8], i11[8], i12[8], i13[8];
    F::sub(i7, x2, x1);
    ld8v(i8, c.item_inv + (size_t)it * 8);    // 1 / i7 (ItemInvTask)
    F::sub(i9, y2, y1);
    F::mul(i10, i8, i9);
    F::sqr(i11, i10);
    F::sub(i12, x1, x3);
    F::mul(i13, i10, i12);
    // derived blinders: C7 = C2 - C1, C9 = C5 - C4, C12 = C1 - C3 (pointAdd.ts:137,139,142)
    uint32_t r7[8], r9[8], r12[8], rcx[8], rcy[8];
    F::sub(r7, mPkx, mT1x);
    F::sub(r9, mPky, mT1y);
    F::sub(r12, mT1x, mTx);
    F::add(rcx, mTx, mT1x); F::add(rcx, rcx, mPkx);   // Cint = C3 + C1 + C2 (pointAdd.ts:151)
    F::add(rcy, mTy, mT1y);                           // Cint = C6 + C4      (pointAdd.ts:158)
    uint32_t r8[8], r10[8], r11[8], r13[8], m8[8], m10[8], m11[8], m13[8];
    draw_checked<FpP256>(r8, c, b, d0 + IT_C8_R);
    draw_checked<FpP256>(r10, c, b, d0 + IT_C10_R);
    draw_checked<FpP256>(r11, c, b, d0 + IT_C11_R);
    draw_checked<FpP256>(r13, c, b, d0 + IT_C13_R);
    F::to_mont(m8, r8); F::to_mont(m10, r10); F::to_mont(m11, r11); F::to_mont(m13, r13);
    job(it, JOB_T1X, x1, rT1x);
    job(it, JOB_T1Y, y1, rT1y);
    job(it, JOB_C8, i8, r8);
    job(it, JOB_C10, i10, r10);
    job(it, JOB_C11, i11, r11);
    job(it, JOB_C13, i13, r13);
    uint32_t one[8], zero[8];
    F::set_one(one);
    zero_n<8>(zero);
    uint32_t* sec = c.secrets + (size_t)it * SECRETS_PER_ITEM * 8;
    // the four MultProofs (pointAdd.ts:145-149,156): (x, y, z, rx, ry, rz)
    for (int m = 0; m < 4; m++) {
      const uint32_t *x, *y, *z, *rx, *ry, *rz;
      if (m == 0)      { x = i7;  y = i8;  z = one; rx = r7;  ry = m8;  rz = zero; }
      else if (m == 1) { x = i8;  y = i9;  z = i10; rx = m8;  ry = r9;  rz = m10; }
      else if (m == 2) { x = i10; y = i10; z = i11; rx = m10; ry = m10; rz = m11; }
      else             { x = i10; y = i12; z = i13; rx = m10; ry = r12; rz = m13; }
      const int dm = d0 + item_mult_draw(m), j0 = JOB_MULT0 + 6 * m;
      uint32_t r4[8];
      mult_openings([&](int k, const uint32_t* v, const uint32_t* r) { job_raw(it, j0 + k, v, r); },
                    [&](int q, uint32_t* r) { draw_checked<FpP256>(r, c, b, dm + q); }, x, y, ry, r4);
      uint32_t* sm = sec + (size_t)m * 7 * 8;
      st8v(sm, x); st8v(sm + 8, y); st8v(sm + 16, z);
      st8v(sm + 24, rx); st8v(sm + 32, ry); st8v(sm + 40, rz); st8v(sm + 48, r4);
    }
    // the two EqualityProofs (pointAdd.ts:151-160): (x, r1, r2)
    for (int e = 0; e < 2; e++) {
      const int de = d0 + (e == 0 ? IT_EQ0 : IT_EQ1), j0 = JOB_EQ0 + 2 * e;
      equality_openings([&](int k, const uint32_t* v, const uint32_t* r) { job_raw(it, j0 + k, v, r); },
                        [&](int q, uint32_t* r) { draw_checked<FpP256>(r, c, b, de + q); });
      uint32_t* se = sec + (size_t)(28 + 3 * e) * 8;
      st8v(se, e == 0 ? i11 : i13);
      st8v(se + 8, e == 0 ? m11 : m13);
      st8v(se + 16, e == 0 ? rcx : rcy);
    }
  }
};

// Stage 6b — derived commitments by point addition (pointAdd.ts:137-159). One thread per item.
struct DerivedTask {
  ProveCtx c;
  struct Store {   // derived point d of item `it`, projective (the address is formed at each store)
    const ProveCtx& c;
    int it;
    ZK_HD void operator()(int d, const TomPt& p) const { tom_st_xyz(c.s2_proj + c.s2_der(it, d) * TOM_E2_WORDS, p.x, p.y, p.z); }
  };
  ZK_HD void ldaff(TomPt& p, const uint32_t* aff, size_t idx) const {
    uint32_t x[PGL], y[PGL];
    ld<PGL>(x, aff + idx * TOM_AFF_WORDS);
    ld<PGL>(y, aff + idx * TOM_AFF_WORDS + PGL);
    tom_from_affine(p, x, y);
  }
  ZK_HD void operator()(int it) const {
    const int b = c.item_b[it], i = c.item_i[it];
    TomPt pkX, pkY, Tx, Ty, T1x, T1y;
    ldaff(pkX, c.s1_aff, c.s1_pt(b, 0));
    ldaff(pkY, c.s1_aff, c.s1_pt(b, 1));
    ldaff(Tx, c.s1_aff, c.s1_pt(b, 2 + 2 * i));
    ldaff(Ty, c.s1_aff, c.s1_pt(b, 3 + 2 * i));
    ldaff(T1x, c.s2_aff, c.s2_job(it, JOB_T1X));
    ldaff(T1y, c.s2_aff, c.s2_job(it, JOB_T1Y));
    // statement of the repetition's PointAddProof: C1..C6 = T1x pkX Tx T1y pkY Ty (exp.ts:199-210)
    point_add_derived(Store{c, it}, T1x, pkX, Tx, T1y, pkY, Ty);
  }
};

// Stage 7 — the six Fiat-Shamir challenges of one item (mult.ts:116, equality.ts:69).
// One thread per (item, h).
struct ItemHashTask {
  ProveCtx c;
  struct Src {
    const ProveCtx* c;
    size_t it;
    int h;
    ZK_HD const uint8_t* pt(size_t idx) const { return c->s2_bytes + idx * BSTRIDE; }
    ZK_HD const uint8_t* operator()(int k, int& len) const {
      len = WP;
      const ProveCtx& C = *c;
      const int ns = h < PA_MULTS ? 3 : 2;   // the statement (zk_sigma.cuh wiring), then the sub-proof's own points
      if (k < ns) {
        const int com = h < PA_MULTS ? pa_mult_com(h, k) : pa_eq_com(h - PA_MULTS, k);
        return pa_com_bytes(com, pt(C.s2_der(it, 0)), C.tg_bytes, pt(C.s2_job(it, JOB_C8)), BSTRIDE);
      }
      return pt(C.s2_job(it, (h < PA_MULTS ? JOB_MULT0 + 6 * h : JOB_EQ0 + 2 * (h - PA_MULTS)) + (k - ns)));
    }
  };
  ZK_HD void operator()(int t) const {
    const size_t it = (size_t)t / HASHES_PER_ITEM;
    const int h = t % HASHES_PER_ITEM;
    uint32_t c3[3];
    Src src{&c, it, h};
    hash_points80(c3, src, h < 4 ? 9 : 4);
    st<3>(c.item_chal + (size_t)t * 3, c3);
  }
};

// Stage 8 — responses + byte assembly of one 0-bit repetition (exp.ts:212-225,
// pointAdd.ts:162, mult.ts:122-130, equality.ts:73-77).  One thread per (item, part):
// part 0..3 MultProof m, 4..5 EqualityProof e, 6 repetition header/tail.  Each part writes its
// contiguous byte regions through one ByteWriter each (a MultProof, an EqualityProof, z z2 C8 C10 C11 C13,
// r1 r2), so neighbouring parts only share the edge blocks of their regions.
struct ItemEmitTask {
  ProveCtx c;
  ZK_HD void operator()(int t) const {
    const size_t it = (size_t)t / 7;
    const int part = t % 7;
    const int b = c.item_b[it], i = c.item_i[it], k = c.item_k[it];
    uint8_t* rep = c.proofs + (size_t)b * c.proof_stride + c.rep_off[(size_t)b * c.S + i];
    uint8_t* body = rep + REP_HEAD;            // z z2 PointAddProof r1 r2
    uint8_t* pa = body + 2 * NS;
    const int d0 = draws_before_items(c.S) + DRAWS_PER_ITEM * k;
    const uint32_t* sec = c.secrets + it * SECRETS_PER_ITEM * 8;
    if (part < 4) {
      const int m = part;
      ByteWriter o(pa + 4 * WP + m * MULT_LEN);
#pragma unroll
      for (int p = 0; p < 6; p++) o.put_point<WP>(c.s2_bytes + c.s2_job(it, JOB_MULT0 + 6 * m + p) * BSTRIDE);
      uint32_t cc[8], c3[3];
      ld<3>(c3, c.item_chal + (it * HASHES_PER_ITEM + m) * 3);
      challenge_to_limbs(cc, c3);
      const uint32_t* sm = sec + (size_t)m * 7 * 8;   // x y z rx ry rz r4
      sigma_responses<7>(o, cc, c.tape_of(b), d0 + item_mult_draw(m), [&](int q, uint32_t* w) { ld8v(w, sm + q * 8); });
      o.finish();
    } else if (part < 6) {
      const int e = part - 4;
      ByteWriter o(pa + 4 * WP + 4 * MULT_LEN + e * EQ_LEN);
      o.put_point<WP>(c.s2_bytes + c.s2_job(it, JOB_EQ0 + 2 * e) * BSTRIDE);
      o.put_point<WP>(c.s2_bytes + c.s2_job(it, JOB_EQ0 + 2 * e + 1) * BSTRIDE);
      uint32_t cc[8], c3[3];
      ld<3>(c3, c.item_chal + (it * HASHES_PER_ITEM + 4 + e) * 3);
      challenge_to_limbs(cc, c3);
      const uint32_t* se = sec + (size_t)(28 + 3 * e) * 8;   // x, C1.r, C2.r
      sigma_responses<3>(o, cc, c.tape_of(b), d0 + (e == 0 ? IT_EQ0 : IT_EQ1), [&](int q, uint32_t* w) { ld8v(w, se + q * 8); });
      o.finish();
    } else {
      // z = alpha - s1, z2 = r_i - comS1.r  (mod n)  (exp.ts:186,221); r1 = T1x.r, r2 = T1y.r
      using Fn = P256n;
      uint32_t alpha[8], s1[8], ri[8], r0[8], z[8];
      tape_draw(alpha, c.tape_of(b), DRAW_REP0 + DRAWS_PER_REP * i); reduce_once<FnP256>(alpha);
      tape_draw(ri, c.tape_of(b), DRAW_REP0 + DRAWS_PER_REP * i + 1); reduce_once<FnP256>(ri);
      tape_draw(r0, c.tape_of(b), DRAW_COMS1_R); reduce_once<FnP256>(r0);
      ld<8>(s1, c.s1 + (size_t)b * 8);
      ByteWriter o(body);                      // z z2 C8 C10 C11 C13
      Fn::sub(z, alpha, s1);
      o.put_scalar<NS>(z);
      Fn::sub(z, ri, r0);
      o.put_scalar<NS>(z);
      o.put_point<WP>(c.s2_bytes + c.s2_job(it, JOB_C8) * BSTRIDE);
      o.put_point<WP>(c.s2_bytes + c.s2_job(it, JOB_C10) * BSTRIDE);
      o.put_point<WP>(c.s2_bytes + c.s2_job(it, JOB_C11) * BSTRIDE);
      o.put_point<WP>(c.s2_bytes + c.s2_job(it, JOB_C13) * BSTRIDE);
      o.finish();
      ByteWriter ot(pa + PA_LEN);              // r1 r2
      uint32_t r[8];
      tape_draw(r, c.tape_of(b), d0 + IT_T1X_R); reduce_once<FpP256>(r);
      ot.put_scalar<WS>(r);
      tape_draw(r, c.tape_of(b), d0 + IT_T1Y_R); reduce_once<FpP256>(r);
      ot.put_scalar<WS>(r);
      ot.finish();
    }
  }
};

// Stage 8b — proof header and per-repetition heads/1-bit bodies.  One thread per (proof, slot),
// slot in [0, S] (slot S writes the 264-byte header R comS1 keyXcom keyYcom).  A 0-bit repetition's
// head is one byte region (its body is ItemEmitTask's), a 1-bit repetition is one region as a whole.
struct RepEmitTask {
  ProveCtx c;
  ZK_HD void operator()(int t) const {
    const int S1 = c.S + 1;
    const int b = t / S1, i = t % S1;
    uint8_t* proof = c.proofs + (size_t)b * c.proof_stride;
    if (i == c.S) {
      if (c.mode == 1) return;   // proveExp alone: the row holds the repetitions only
      ByteWriter o(proof);
      o.put_point<NP>(c.r_bytes + (size_t)b * BSTRIDE);
      o.put_point<NP>(c.pa_A_bytes + ((size_t)b * S1 + c.S) * BSTRIDE);
      o.put_point<WP>(c.s1_bytes + c.s1_pt(b, 0) * BSTRIDE);
      o.put_point<WP>(c.s1_bytes + c.s1_pt(b, 1) * BSTRIDE);
      o.finish();
      if (c.pa_A_inf[(size_t)b * S1 + c.S]) ZK_SET_STATUS(c.status + b, ZKA_ERR_IDENTITY_ENC);
      return;
    }
    uint8_t* rep = proof + c.rep_off[(size_t)b * c.S + i];
    const uint32_t bit = (c.chal[(size_t)b * 3 + (i >> 5)] >> (i & 31)) & 1u;
    ByteWriter o(rep);
    o.put_byte(bit);
    o.put_point<NP>(c.pa_A_bytes + ((size_t)b * S1 + i) * BSTRIDE);
    o.put_point<WP>(c.s1_bytes + c.s1_pt(b, 2 + 2 * i) * BSTRIDE);
    o.put_point<WP>(c.s1_bytes + c.s1_pt(b, 3 + 2 * i) * BSTRIDE);
    if (bit) {   // exp.ts:170-183: alpha, r, Tx.r, Ty.r
      uint32_t r[8];
#pragma unroll
      for (int q = 0; q < 4; q++) {
        tape_draw(r, c.tape_of(b), DRAW_REP0 + DRAWS_PER_REP * i + q);
        if (q < 2) { reduce_once<FnP256>(r); o.put_scalar<NS>(r); }
        else       { reduce_once<FpP256>(r); o.put_scalar<WS>(r); }
      }
    }
    o.finish();
  }
};

// ---------------------------------------------------------------------------------------------
// Groth-Kohlweiss membership (gk.ts:94-195), scalar variant over the ring of key x-coordinates.
// ---------------------------------------------------------------------------------------------
ZK_HD int gk_draw0(const ProveCtx& c, int b) { return draws_before_items(c.S) + DRAWS_PER_ITEM * (int)c.zcount[b]; }

// jobs cl_i = commit(l_i, r_i), ca_i = commit(a_i, s_i), cb_i = commit(l_i a_i, t_i) (gk.ts:129-133)
// One thread per (proof, i).
struct GkJobsTask {
  ProveCtx c;
  ZK_HD void operator()(int t) const {
    const int b = t / c.n, i = t % c.n, n = c.n_row(b);
    uint32_t ri[8], ai[8], si[8], ti[8], v[8];
    if (i >= n) {   // beyond the row's depth: the thread zeroes four of the row's unused slots [4 n, 4 c.n)
      zero_n<8>(v);
      for (int q = 0; q < 4; q++) {
        const size_t j = c.s2_gk(b, 4 * i + q);
        st8v(c.s2_jv + j * 8, v); st8v(c.s2_jr + j * 8, v);
      }
      return;
    }
    const int d = gk_draw0(c, b) + DRAWS_PER_GK_ROUND * i;
    draw_checked<FpP256>(ri, c, b, d + 0);
    draw_checked<FpP256>(ai, c, b, d + 1);
    draw_checked<FpP256>(si, c, b, d + 2);
    draw_checked<FpP256>(ti, c, b, d + 3);
    const uint32_t bit = (c.which_s[b] >> i) & 1u;
    zero_n<8>(v);
    v[0] = bit;
    size_t j = c.s2_gk(b, i);                        // cl_i
    st8v(c.s2_jv + j * 8, v); st8v(c.s2_jr + j * 8, ri);
    j = c.s2_gk(b, n + i);                           // ca_i
    st8v(c.s2_jv + j * 8, ai); st8v(c.s2_jr + j * 8, si);
    j = c.s2_gk(b, 2 * n + i);                       // cb_i
    if (bit) copy_n<8>(v, ai); else zero_n<8>(v);
    st8v(c.s2_jv + j * 8, v); st8v(c.s2_jr + j * 8, ti);
  }
};

// d(omega_w) = sum_i (v_which - v_i) * prod_j (bit_j(i) ? f1j : f0j)   (gk.ts:141-171),
// f0j = (1-l_j) w - a_j, f1j = l_j w + a_j.  One thread per (proof, w); O(3 * 2^n) modmuls,
// products maintained incrementally over the binary counter (no inversions, no p[] array).
// If some f0j == 0 the reference's ratio trick yields dval = 0 (invMod(0) = 0); reproduced.
struct GkPolyTask {     // one thread per (proof, w, ring block)
  ProveCtx c;
  ZK_HD void operator()(int t) const {
    using F = Tomq;
    const int gblk = 1 << (c.n - gk_block_bits(c.n));   // the grid: c.n points w and gblk blocks per proof
    const int blk = t % gblk, bw = t / gblk;
    const int b = bw / c.n, w = bw % c.n;
    const int n = c.n_row(b), k = gk_block_bits(n);
    const int nblk = 1 << (n - k);
    if (w >= n || blk >= nblk) return;
    const int d0 = gk_draw0(c, b);
    uint32_t f0[20][8], f1[20][8];
    uint32_t wm[8], wc[8];
    zero_n<8>(wc);
    wc[0] = (uint32_t)w;
    F::to_mont(wm, wc);
    bool degenerate = false;
    for (int j = 0; j < n; j++) {
      uint32_t a[8], am[8];
      draw_checked<FpP256>(a, c, b, d0 + DRAWS_PER_GK_ROUND * j + 1);
      F::to_mont(am, a);
      const uint32_t bit = (c.which_s[b] >> j) & 1u;
      if (bit) { F::neg(f0[j], am); F::add(f1[j], wm, am); }
      else     { F::sub(f0[j], wm, am); copy_n<8>(f1[j], am); }
      if (is_zero_n<8>(f0[j])) degenerate = true;
    }
    uint32_t dval[8], vw[8];
    zero_n<8>(dval);
    const uint32_t* ring = c.ring_of_row(b);
    ld<8>(vw, ring + (size_t)c.which_s[b] * 8);
    if (!degenerate) gk_block_sum(dval, ring, f0, f1, n, k, (uint32_t)blk, vw);
    uint32_t* out = nblk == 1 ? c.gk_dv + (size_t)bw * 8 : c.gk_part + (size_t)t * 8;
    st<8>(out, dval);
  }
};
struct GkPolyReduceTask {   // d(omega_w) = sum of the block sums (only launched when n > GK_BLOCK_BITS)
  ProveCtx c;
  ZK_HD void operator()(int bw) const {
    using F = Tomq;
    const int gblk = 1 << (c.n - gk_block_bits(c.n));
    const int n = c.n_row(bw / c.n), nblk = 1 << (n - gk_block_bits(n));
    if (bw % c.n >= n || nblk == 1) return;   // no such point, or GkPolyTask wrote gk_dv itself
    uint32_t acc[8], v[8];
    zero_n<8>(acc);
    for (int i = 0; i < nblk; i++) {
      ld<8>(v, c.gk_part + ((size_t)bw * gblk + i) * 8);
      F::add(acc, acc, v);
    }
    st<8>(c.gk_dv + (size_t)bw * 8, acc);
  }
};

// Lagrange matrix for nodes 0..n-1 mod q (interpolate.ts:27-70): coeff_j = sum_i L[j][i] y_i.
// One thread, once per call.
struct GkLagrangeTask {
  uint32_t* lag;  // [n][n][8] Montgomery
  int n;
  ZK_HD void operator()(int) const {
    using F = Tomq;
    uint32_t s[21][8];
    uint32_t xs[20][8];
    for (int i = 0; i < n; i++) {
      uint32_t cidx[8];
      zero_n<8>(cidx);
      cidx[0] = (uint32_t)i;
      F::to_mont(xs[i], cidx);
    }
    for (int i = 0; i <= n; i++) zero_n<8>(s[i]);
    // s(x) = prod (x - x_i)
    F::set_one(s[n]);
    F::neg(s[n - 1], xs[0]);
    for (int i = 1; i < n; i++) {
      for (int j = n - i - 1; j < n - 1; j++) {
        uint32_t t[8];
        F::mul(t, xs[i], s[j + 1]);
        F::sub(s[j], s[j], t);
      }
      F::sub(s[n - 1], s[n - 1], xs[i]);
    }
    for (int i = 0; i < n; i++) {
      // phi = s'(x_i)
      uint32_t phi[8], ff[8];
      zero_n<8>(phi);
      for (int j = n; j >= 1; j--) {
        uint32_t jm[8], jc[8], t[8];
        zero_n<8>(jc);
        jc[0] = (uint32_t)j;
        F::to_mont(jm, jc);
        F::mul(t, jm, s[j]);
        F::mul(phi, phi, xs[i]);
        F::add(phi, phi, t);
      }
      F::inv(ff, phi);
      uint32_t bb[8];
      F::set_one(bb);
      for (int j = n - 1; j >= 0; j--) {
        uint32_t t[8];
        F::mul(t, bb, ff);
        st<8>(lag + ((size_t)j * n + i) * 8, t);
        F::mul(t, xs[i], bb);
        F::add(bb, s[j], t);
      }
    }
  }
};

// the matrices of the depths 1..count for a ring set, depth d at word ProveCtx::gk_lag_off(d).  One thread per depth.
struct GkLagrangeSetTask {
  uint32_t* lag;
  ZK_HD void operator()(int t) const { GkLagrangeTask{lag + ProveCtx::gk_lag_off(t + 1), t + 1}(0); }
};

// cd_k = commit(d_k, rho_k), d = L * dv  (gk.ts:173-176).  One thread per (proof, k).
struct GkCdJobsTask {
  ProveCtx c;
  ZK_HD void operator()(int t) const {
    using F = Tomq;
    const int b = t / c.n, k = t % c.n, n = c.n_row(b);
    if (k >= n) return;
    const uint32_t* lag = c.gk_lag_row(b);
    uint32_t acc[8];
    zero_n<8>(acc);
    for (int i = 0; i < n; i++) {
      uint32_t l[8], y[8], m[8];
      ld<8>(l, lag + ((size_t)k * n + i) * 8);
      ld<8>(y, c.gk_dv + ((size_t)b * c.n + i) * 8);
      F::mul(m, l, y);
      F::add(acc, acc, m);
    }
    uint32_t v[8], rho[8];
    F::from_mont(v, acc);
    draw_checked<FpP256>(rho, c, b, gk_draw0(c, b) + DRAWS_PER_GK_ROUND * k + 4);
    const size_t j = c.s2_gk(b, 3 * n + k);
    st<8>(c.s2_jv + j * 8, v);
    st<8>(c.s2_jr + j * 8, rho);
  }
};

// x = H(cl, ca, cb, cd) (gk.ts:179-180), responses (gk.ts:184-192) and GK bytes.  Per proof.
struct GkEmitTask {
  ProveCtx c;
  struct Src {
    const ProveCtx* c;
    int b;
    ZK_HD const uint8_t* operator()(int k, int& len) const {
      len = WP;
      return c->s2_bytes + c->s2_gk(b, k) * BSTRIDE;
    }
  };
  ZK_HD void operator()(int b) const {
    using F = Tomq;
    const int n = c.n_row(b);
    uint32_t c3[3], xc[8], xm[8];
    Src src{&c, b};
    hash_points80(c3, src, 4 * n);
    st<3>(c.gk_x + (size_t)b * 3, c3);
    challenge_to_limbs(xc, c3);
    F::to_mont(xm, xc);
    // byte regions: n and the 4n points, then the f, za and zb arrays (zd follows zb)
    uint8_t* o = c.proofs + (size_t)b * c.proof_stride + c.gk_off[b];
    {
      ByteWriter op(o);
      op.put_byte((uint32_t)n);
      for (int k = 0; k < 4 * n; k++) op.put_point<WP>(c.s2_bytes + c.s2_gk(b, k) * BSTRIDE);
      op.finish();
    }
    o += 1 + (size_t)4 * n * WP;
    ByteWriter of(o), oza(o + (size_t)n * WS), ozb(o + (size_t)2 * n * WS);
    const int d0 = gk_draw0(c, b);
    uint32_t zd[8], xp[8], t[8], u[8];
    // zd = pkX.r * x^n - sum rho_i x^i
    F::set_one(xp);
    zero_n<8>(zd);
    for (int i = 0; i < n; i++) {
      uint32_t ri[8], ai[8], si[8], ti[8], rho[8];
      tape_draw(ri, c.tape_of(b), d0 + 5 * i + 0); reduce_once<FpP256>(ri);
      tape_draw(ai, c.tape_of(b), d0 + 5 * i + 1); reduce_once<FpP256>(ai);
      tape_draw(si, c.tape_of(b), d0 + 5 * i + 2); reduce_once<FpP256>(si);
      tape_draw(ti, c.tape_of(b), d0 + 5 * i + 3); reduce_once<FpP256>(ti);
      tape_draw(rho, c.tape_of(b), d0 + 5 * i + 4); reduce_once<FpP256>(rho);
      const uint32_t bit = (c.which_s[b] >> i) & 1u;
      // f_i = l_i x + a_i
      uint32_t f[8];
      if (bit) F::add(f, xc, ai); else copy_n<8>(f, ai);
      of.put_scalar<WS>(f);
      // za_i = r_i x + s_i
      F::mul(t, ri, xm);          // canonical r_i * x
      F::add(u, t, si);
      oza.put_scalar<WS>(u);
      // zb_i = r_i (x - f_i) + t_i
      F::sub(u, xc, f);
      F::to_mont(u, u);
      F::mul(t, ri, u);
      F::add(u, t, ti);
      ozb.put_scalar<WS>(u);
      // zd -= rho_i x^i   (xp = x^i in Montgomery form)
      F::mul(t, rho, xp);
      F::sub(zd, zd, t);
      F::mul(xp, xp, xm);
    }
    uint32_t rpk[8];
    tape_draw(rpk, c.tape_of(b), DRAW_PKX_R); reduce_once<FpP256>(rpk);
    F::mul(t, rpk, xp);           // pkX.r * x^n
    F::add(zd, zd, t);
    ozb.put_scalar<WS>(zd);
    of.finish();
    oza.finish();
    ozb.finish();
  }
};

// proveExp alone: the statement  s*g - Q = P  is an input here, not something the pipeline constructed.  Phase B
// evaluates T1 = T_i - P, which equals the reference's g*z + Q exactly when the statement holds; otherwise the
// reference throws "Points don't add up!" in provePointAdd (pointAdd.ts:104-106).  Slot S of phase A is s*g.
struct ExpStatementTask {
  ProveCtx c;
  ZK_HD void operator()(int b) const {
    using F = P256p;
    const size_t slot = (size_t)b * (c.S + 1) + c.S;
    P256Aff sg, q, pk;
    p256_ld_aff(sg, c.pa_T_aff + slot * 16);
    p256_ld_aff(pk, c.pk_aff + (size_t)b * 16);
    P256Pt acc;
    if (c.pa_T_inf[slot]) p256_set_identity(acc); else p256_from_affine(acc, sg);
    if (!c.q_inf[b]) {
      p256_ld_aff(q, c.q_aff + (size_t)b * 16);
      F::neg(q.y, q.y);
      p256_madd(acc, acc, q);
    }
    F::neg(pk.y, pk.y);
    p256_madd(acc, acc, pk);          // s*g - Q - P
    if (!p256_is_identity(acc)) ZK_SET_STATUS(c.status + b, ZKA_ERR_POINTS_DONT_ADD);
  }
};

// proveMembership alone: per-proof setup of the pieces the GK tasks expect from the full pipeline.  The internal
// tape row is [0, com.r, 0] followed by the caller's 5n draws (with S = 0 the GK draws start at index 3).
struct GkAloneSetupTask {
  ProveCtx c;
  const uint8_t* com_r;    // [B][32]
  const uint8_t* tape;     // [B][tape_stride]
  size_t tape_stride;
  uint8_t* itape;          // [B][c.tape_stride]: 96 + tape_stride rounded up to a multiple of 16
  ZK_HD void operator()(int b) const {
    c.status[b] = ZKA_OK;
    c.zcount[b] = 0;
    c.gk_off[b] = 0;
    c.proof_len[b] = (uint32_t)gk_len(c.n);
    const uint32_t w = c.which[b];
    const uint32_t nr = c.ring_size_row(b);
    c.which_s[b] = w < nr ? w : 0u;
    if (w >= nr) ZK_SET_STATUS(c.status + b, ZKA_ERR_BAD_INDEX);
    uint8_t* row = itape + (size_t)b * c.tape_stride;
    for (int i = 0; i < 96; i++) row[i] = (i >= 32 && i < 64) ? com_r[(size_t)b * 32 + (i - 32)] : 0;
    const size_t need = (size_t)32 * 5 * c.n;
    for (size_t i = 0; i < need; i++) row[96 + i] = tape[(size_t)b * tape_stride + i];
    uint32_t r[8];
    tape_draw(r, com_r + (size_t)b * 32, 0);   // = draw DRAW_PKX_R of the row (not read back: the row is written here)
    if (!lt_p<FpP256>(r)) ZK_SET_STATUS(c.status + b, ZKA_ERR_TAPE_RANGE);
  }
};

// ---- proveEquality / proveMult alone (equality.ts:60-78, mult.ts:93-131) ---------------------------------------
// The statement's commitments are given by their openings; every point of the proof is a commitment with a known
// opening, so all of them are jobs of the fixed-base commitment kernel.
//   equality: scalars = x r1 r2,       draws = k A1.r A2.r,                    jobs = C1 C2 A1 A2
//   mult:     scalars = x y z rx ry rz, draws = k_x k_y k_z Ax.r Ay.r Az.r A4_1.r, jobs = Cx Cy Cz C4 Ax Ay Az A4_1 A4_2
enum : int { SUBP_EQ_JOBS = 4, SUBP_MULT_JOBS = 9 };
struct SubProveJobsTask {
  int kind;                 // 0 equality, 1 mult
  const uint8_t* scalars;   // [B][3|6][32]
  const uint8_t* tape;      // [B][tape_stride]
  size_t tape_stride;
  uint32_t *jv, *jr;        // [B][4|9][8]
  int32_t* status;
  ZK_HD static bool rd(uint32_t* r, const uint8_t* p, int draw = 0) {   // draw `draw` of the row at p
    tape_draw(r, p, draw);
    if (lt_p<FpP256>(r)) return true;
    sub_p<FpP256>(r, r);
    return false;
  }
  ZK_HD void operator()(int b) const {
    using F = Tomq;
    status[b] = ZKA_OK;
    const uint8_t* sc = scalars + (size_t)b * (kind == 0 ? 3 : 6) * 32;
    const uint8_t* dr = tape + (size_t)b * tape_stride;
    const int J = kind == 0 ? SUBP_EQ_JOBS : SUBP_MULT_JOBS;
    uint32_t* v = jv + (size_t)b * J * 8;
    uint32_t* r = jr + (size_t)b * J * 8;
    bool ok = true;
    const int j0 = kind == 0 ? 2 : 3;   // the proof's own points follow the statement's
    auto job = [&](int k, const uint32_t* vk, const uint32_t* rk) { st<8>(v + 8 * (j0 + k), vk); st<8>(r + 8 * (j0 + k), rk); };
    auto draw = [&](int q, uint32_t* d) { ok = rd(d, dr, q) && ok; };
    if (kind == 0) {
      uint32_t x[8], r1[8], r2[8];
      rd(x, sc); rd(r1, sc + 32); rd(r2, sc + 64);      // newScalar reduces the statement's values
      st<8>(v, x); st<8>(r, r1); st<8>(v + 8, x); st<8>(r + 8, r2);
      equality_openings(job, draw);
    } else {
      uint32_t s[6][8];   // x y z rx ry rz
      for (int q = 0; q < 6; q++) rd(s[q], sc + 32 * q);
      for (int k = 0; k < 3; k++) { st<8>(v + 8 * k, s[k]); st<8>(r + 8 * k, s[3 + k]); }
      uint32_t xm[8], ym[8], rym[8], r4[8];
      F::to_mont(xm, s[0]); F::to_mont(ym, s[1]); F::to_mont(rym, s[4]);
      mult_openings(job, draw, xm, ym, rym, r4);
    }
    if (!ok) ZK_SET_STATUS(status + b, ZKA_ERR_TAPE_RANGE);
  }
};
struct SubProveEmitTask {
  int kind;
  const uint8_t* scalars;
  const uint8_t* tape;
  size_t tape_stride;
  const uint32_t* jr;       // [B][J][8] (r4 = x*ry is job 3's blinder)
  const uint8_t* bytes;     // [B][J][BSTRIDE] encodings of the jobs
  uint8_t* commitments;     // [B][2|3][67]
  uint8_t* proofs;          // [B][233|633]
  int32_t* status;
  ZK_HD void operator()(int b) const {
    using F = Tomq;
    const int J = kind == 0 ? SUBP_EQ_JOBS : SUBP_MULT_JOBS, nc = kind == 0 ? 2 : 3, plen = kind == 0 ? EQ_LEN : MULT_LEN;
    uint8_t* out = proofs + (size_t)b * plen;
    uint8_t* com = commitments + (size_t)b * nc * WP;
    if (status[b] != ZKA_OK) {
      for (int i = 0; i < plen; i++) out[i] = 0;
      for (int i = 0; i < nc * WP; i++) com[i] = 0;
      return;
    }
    const uint8_t* pb = bytes + (size_t)b * J * BSTRIDE;
    const uint8_t* sc = scalars + (size_t)b * (kind == 0 ? 3 : 6) * 32;
    const uint8_t* dr = tape + (size_t)b * tape_stride;
    uint32_t c3[3], cc[8];   // the challenge hashes the statement, then the proof's own points: every job in order
    hash_points80(c3, [&](int j, int& len) { len = WP; return pb + (size_t)j * BSTRIDE; }, J);
    challenge_to_limbs(cc, c3);
    ByteWriter oc(com), o(out);
    for (int j = 0; j < nc; j++) oc.put_point<WP>(pb + (size_t)j * BSTRIDE);
    oc.finish();
    for (int j = nc; j < J; j++) o.put_point<WP>(pb + (size_t)j * BSTRIDE);
    // the secrets are the statement's scalars in row order, then (mult) r4 = x ry, the blinder of C4 (job 3)
    auto w = [&](int q, uint32_t* wm) {
      uint32_t s[8];
      if (q < 6) { limbs_from_be<8>(s, sc + 32 * q, 32); reduce_once<FpP256>(s); }
      else ld<8>(s, jr + ((size_t)b * J + 3) * 8);
      F::to_mont(wm, s);
    };
    if (kind == 0) sigma_responses<3>(o, cc, dr, 0, w);
    else sigma_responses<7>(o, cc, dr, 0, w);
    o.finish();
  }
};

// ---- provePointAdd alone (pointAdd.ts:92-163): one statement = one "item" of the batched prover ------------------
// The stage tasks of a 0-bit repetition are reused with S = 1: T1 := P, pk := Q, T_0 := R.  Internal tape row:
//   [0, QX.r, QY.r, 0, 0, RX.r, RY.r, PX.r, PY.r, the caller's 38 draws].
struct PaddSetupTask {
  ProveCtx c;
  const uint8_t* points;    // [B][3][65] P Q R
  const uint8_t* blinders;  // [B][6][32] PX.r PY.r QX.r QY.r RX.r RY.r
  const uint8_t* tape;      // [B][tape_stride] 38 draws
  size_t tape_stride;
  uint8_t* itape;           // [B][c.tape_stride]
  ZK_HD void operator()(int b) const {
    c.status[b] = ZKA_OK;
    P256Aff P, Q, R;
    bool infP, infQ, infR;
    const uint8_t* pb = points + (size_t)b * 3 * 65;
    const bool okP = p256_parse(P, infP, pb), okQ = p256_parse(Q, infQ, pb + 65), okR = p256_parse(R, infR, pb + 130);
    if (!okP || !okQ || !okR || infP || infQ || infR) {   // not on the curve, or 'P/Q/R is at infinity' (pointAdd.ts:113-124)
      ZK_SET_STATUS(c.status + b, ZKA_ERR_INVALID_PK);
      p256_set_generator(P); p256_set_generator(Q); p256_set_generator(R);
    } else {
      P256Pt s, nr;
      p256_from_affine(s, P);
      p256_madd(s, s, Q);
      P256Aff n = R;
      P256p::neg(n.y, n.y);
      p256_madd(nr, s, n);
      if (!p256_is_identity(nr)) ZK_SET_STATUS(c.status + b, ZKA_ERR_POINTS_DONT_ADD);   // pointAdd.ts:104-106
    }
    p256_st_aff(c.pb_T1_aff + (size_t)b * 16, P);
    p256_st_aff(c.pk_aff + (size_t)b * 16, Q);
    p256_st_aff(c.pa_T_aff + (size_t)b * 2 * 16, R);
    c.pa_T_inf[(size_t)b * 2] = 0; c.pa_T_inf[(size_t)b * 2 + 1] = 0;
    c.pa_A_inf[(size_t)b * 2] = 0; c.pa_A_inf[(size_t)b * 2 + 1] = 0;
    c.pb_T1_inf[b] = 0;
    c.chal[(size_t)b * 3] = 0; c.chal[(size_t)b * 3 + 1] = 0; c.chal[(size_t)b * 3 + 2] = 0;
    c.zcount[b] = 1;
    c.item_base[b] = (uint32_t)b;
    c.item_b[b] = (uint32_t)b; c.item_i[b] = 0; c.item_k[b] = 0;
    c.rep_off[b] = 0;
    uint32_t z[8];
    zero_n<8>(z);
    st<8>(c.s1 + (size_t)b * 8, z);
    uint8_t* row = itape + (size_t)b * c.tape_stride;
    const uint8_t* bl = blinders + (size_t)b * 6 * 32;
    const int src[9] = {-1, 2, 3, -1, -1, 4, 5, 0, 1};   // draw index -> blinder index
    for (int d = 0; d < 9; d++)
      for (int i = 0; i < 32; i++) row[32 * d + i] = src[d] < 0 ? 0 : bl[32 * src[d] + i];
    for (int i = 0; i < 32 * 38; i++) row[32 * 9 + i] = tape[(size_t)b * tape_stride + i];
  }
};
struct PaddExtractTask {
  ProveCtx c;
  uint8_t* commitments;     // [B][6][67] PX PY QX QY RX RY
  uint8_t* proofs;          // [B][3266]
  ZK_HD void operator()(int b) const {
    uint8_t* out = proofs + (size_t)b * PA_LEN;
    uint8_t* com = commitments + (size_t)b * 6 * WP;
    if (c.status[b] != ZKA_OK) {
      for (int i = 0; i < PA_LEN; i++) out[i] = 0;
      for (int i = 0; i < 6 * WP; i++) com[i] = 0;
      return;
    }
    const uint8_t* pa = c.proofs + (size_t)b * c.proof_stride + REP_HEAD + 2 * NS;
    for (int i = 0; i < PA_LEN; i++) out[i] = pa[i];
    ByteWriter o(com);
    o.put_point<WP>(c.s2_bytes + c.s2_job(b, JOB_T1X) * BSTRIDE);
    o.put_point<WP>(c.s2_bytes + c.s2_job(b, JOB_T1Y) * BSTRIDE);
    for (int j = 0; j < 4; j++) o.put_point<WP>(c.s1_bytes + c.s1_pt(b, j) * BSTRIDE);
    o.finish();
  }
};

// Last stage: a proof whose status is not ZKA_OK must not leave the library (its blinders may have been
// replaced by zeros or reduced values, which would open the commitments): the row is zeroed and its
// length set to 0.  FIN_PARTS threads per proof, each clears its share of the row with 16-byte stores.
enum : int { FIN_PARTS = 64 };
struct FinalizeTask {
  ProveCtx c;
  ZK_HD void operator()(int t) const {
    const int b = t / FIN_PARTS, part = t % FIN_PARTS;
    if (c.status[b] == ZKA_OK) return;
    uint8_t* row = c.proofs + (size_t)b * c.proof_stride;
    const size_t per = (c.proof_stride + FIN_PARTS - 1) / FIN_PARTS;
    size_t lo = per * part, hi = lo + per;
    if (hi > c.proof_stride) hi = c.proof_stride;
    for (size_t i = lo; i < hi; i++) row[i] = 0;
    if (part == 0) c.proof_len[b] = 0;
  }
};

// ring bytes -> Montgomery residues mod q, padded to 2^n with ring[0] (gk.ts:75-86)
struct RingPrepTask {
  const uint8_t* ring;  // [N][32]
  uint32_t* ring_m;     // [2^n][8]
  int N;
  ZK_HD void operator()(int i) const {
    const int src = i < N ? i : 0;
    uint32_t v[8], m[8];
    limbs_from_be<8>(v, ring + (size_t)src * 32, 32);
    reduce_once<FpP256>(v);
    Tomq::to_mont(m, v);
    st<8>(ring_m + (size_t)i * 8, m);
  }
};

// every ring of a ring set at once: one thread per padded entry i finds its ring r (the last with ring_base[r] <= i) by
// binary search, then converts and pads like RingPrepTask, ring r with its own first entry
struct RingSetPrepTask {
  const uint8_t* keys;         // the rings' 32-byte entries concatenated in ring order
  const uint32_t* key_off;     // [R] first entry of ring r in `keys`
  const uint32_t* ring_base;   // [R] first entry of ring r in ring_m (ring_base[r + 1] - ring_base[r] = 2^n_r)
  const uint32_t* ring_size;   // [R]
  uint32_t* ring_m;            // [total][8]
  int R;
  ZK_HD void operator()(int i) const {
    int lo = 0, hi = R - 1;
    while (lo < hi) {
      const int mid = (lo + hi + 1) >> 1;
      if (ring_base[mid] <= (uint32_t)i) lo = mid; else hi = mid - 1;
    }
    const uint32_t j = (uint32_t)i - ring_base[lo];
    const uint32_t src = key_off[lo] + (j < ring_size[lo] ? j : 0u);
    uint32_t v[8], m[8];
    limbs_from_be<8>(v, keys + (size_t)src * 32, 32);
    reduce_once<FpP256>(v);
    Tomq::to_mont(m, v);
    st<8>(ring_m + (size_t)i * 8, m);
  }
};

}  // namespace zk
