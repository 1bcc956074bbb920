// zk_verify.cuh — stage tasks of the batched verifier (verifySignatureList over B proofs).
//
// Reference call tree being replaced (per proof):
//   /root/reference/src/zkpAttestList.ts:147-184  verifySignatureList (secparam = 20 literal, :177)
//   /root/reference/src/proofGK/gk.ts:197-262     verifyMembership
//   /root/reference/src/exp/exp.ts:233-349        verifyExp  (+ generateIndices :95-109)
//   /root/reference/src/exp/pointAdd.ts:199-259   aggregatePointAdd
//   /root/reference/src/commit/mult.ts:148-175    aggregateMult      (5 relations)
//   /root/reference/src/commit/equality.ts:94-116 aggregateEquality  (2 relations)
//   /root/reference/src/curves/multimult.ts       Relation.drain (one fresh random scalar per
//                                                 relation), MultiMult.evaluate (Bos-Coster heap)
//
// The verifier's decision is `isIdentity()` of three linear combinations (GK, multiW, multiN).
// A linear combination does not depend on how it is evaluated, so the GPU
//   * folds every term on a FIXED base (g, h of both groups, R via its per-proof table, and the
//     recomputed commitments T1x = sx g + r1 h, T1y, C7, C9, C12, Cint which are known
//     combinations of g, h and proof points) into a handful of scalars per proof,
//   * evaluates the remaining variable points (<= 682 tomEdwards256 + 21 P-256 + 4n+1 GK points
//     per proof, 256-bit scalars) with a bucket (Pippenger) MSM, one thread per (proof, window),
// using exactly the reference's randomizers (tape order below), so decisions agree even on
// invalid proofs.
//
// Verifier tape (per proof; include/zkattest.h):
//   [0, 32(2n+1))            GK drains in call order: rel0_0, rel1_0, rel0_1, ... , relFinal  (mod tom.order)
//   [G, G+78)                generateIndices: byte i is rnd(80 - i) already rejection-filtered (< 80 - i)
//   [G+96, ...)              exp drains, packed in consumption order: for each sampled repetition
//                            bit 1: relA (mod p256.n), relTx, relTy (mod tom.order)            = 3 draws
//                            bit 0: relA (mod p256.n), then pi8(5) pi10(5) pi11(5) pix(2) pi13(5) piy(2) = 25 draws
#pragma once
#include "zk_prove.cuh"   // shared item layout, the sigma-protocol layer (zk_sigma.cuh)

namespace zk {

enum : int {
  V_SAMPLES = 20,              // default number of sampled repetitions: the literal secparam of zkpAttestList.ts:177
  V_ENT_PER_SAMPLE = 2 + PA_ENTRIES,   // 34 variable tomEdwards256 points of one sampled 0-bit repetition: Tx, Ty, PointAddProof
  V_SEG = 20,                  // sampled repetitions per MSM segment (one window thread walks <= V_ENT_SEG entries)
  V_ENT_SEG = V_SEG * V_ENT_PER_SAMPLE + 2,       // 682 (+ keyXcom, keyYcom ride with segment 0)
  V_IDX_PAD = 96,
  V_PART_WORDS = 7 * 8,        // per-sample partial sums: gW hW pkX pkY | sR shN sCom
  MSM_C = 6,                   // SIGNED 6-bit bucket windows (tom): digits in [-32, 31], 32 buckets,
  MSM_NWIN = 43,               // 43 windows cover the 258 bits of k + offset (msm_digit6)
  MSM_C_N = 4,                 // P-256 MSM: SIGNED 4-bit windows, digits in [-8, 7], 8 buckets,
  MSM_NWIN_N = 65,             // 65 windows cover the 257 bits of k + offset (msm_digit4)
  // control words of the chunk-wide aggregate check (zk_verify_agg.cuh)
  AGG_SKIP = 0,                // != 0: some proof of the chunk is not eligible, the aggregate kernels return at once
  AGG_TOM_PASS = 1,            // != 0: sum_b (wG_b GK_b + wW_b W_b) is the identity -> the per-proof tomEdwards256 MSMs are skipped
  AGG_NIST_PASS = 2,           // != 0: sum_b wN_b N_b is the identity -> the per-proof P-256 MSMs are skipped
  AGG_CTL_WORDS = 4,
  // the aggregate's weights of a row (zk_verify_agg.cuh): one per combination, in the order of the fixed-base jobs
  // (0: GK, 1: multiW), then multiN
  AGG_W_GK = 0, AGG_W_W = 1, AGG_W_N = 2, AGG_WT = 3,
};

// Status precedence of a row (include/zkattest.h): the reference throws at the first defect it meets, so a row with several
// defects reports that one.  status[] takes, first writer wins (ZK_SET_STATUS, in launch order), what is thrown before
// verifyExp: a proof that does not parse (VLayoutTask, VValidateTask), then R at infinity (VChallengeTask), then a GK draw
// out of range (VReduceTask).  verifyExp's own throws (exp.ts:253-345) come from several kernels, and from concurrent
// threads of one proof, but the reference meets them in sample order: each writer posts a key to vkey[] with
// ZK_POST_MIN and VFinalTask keeps the smallest.  A key is (sample + 1) << 8 | phase << 4 | code, sample -1 being the
// generateIndices draws; inside one sample the phases follow verifyExp: 'params not found', the first draw (relA), T / T1
// at infinity, the later draws.
enum : int { VK_NONE = 0x7fffffff, VK_PARAMS = 0, VK_FIRST_DRAW = 1, VK_T_INF = 2, VK_DRAWS = 3 };
ZK_HD int vkey(int sample, int phase, int code) { return ((sample + 1) << 8) | (phase << 4) | code; }

// K = number of sampled repetitions (verifyExp's secparam, exp.ts:233-262): 20 in verifySignatureList
ZK_LAYOUT_FN size_t verify_tape_len(int n, int /*reps*/, int K = V_SAMPLES) {
  return (size_t)32 * (2 * n + 1) + V_IDX_PAD + (size_t)32 * 25 * K;
}

struct VerifyCtx {
  int B, S, N, n;              // n: the depth the chunk is laid out for (ProveCtx::n); n_row(b) is row b's own
  int K;                       // sampled repetitions (<= S)
  int mode;                    // 0: verifySignatureList; 1: verifyExp alone (exp.ts:233, no GK block, Q given or absent);
                               // 2: verifyMembership alone (gk.ts:197)
  const uint8_t* q_ext;        // mode 1: [B][65] Q points (all-zero = identity) or null (no Q: T1 = g*z)
  FbShape tom;                 // shape of the proof group's two fixed-base tables (g, h)
  const uint8_t* msg_hash;     // [B][32]
  const uint8_t* proofs;       // [B][proof_stride]
  size_t proof_stride;
  const uint32_t* proof_len;   // [B]
  const uint8_t* tape;         // [B][tape_stride]
  size_t tape_stride;
  const uint32_t* ring_m;      // [2^n][8] Montgomery mod q (a ring set: all its rings, see ProveCtx)
  const uint32_t* ring_of;     // [B] ring-set calls: the ring of each row (null: ring_m for every row)
  const uint32_t* ring_base;   // [R] entry offset of each padded ring of the set
  const uint32_t* ring_depth;  // [R] n_r = ceil(log2 N_r) <= n
  const uint32_t* g_tab8;
  const uint32_t* h_tab8;
  int h_w;
  const uint32_t* tg_tab;
  const uint32_t* th_tab;
  const uint8_t* tg_bytes;
  // per proof
  uint32_t* rep_off;    // [B][S]
  uint32_t* gk_off;     // [B]
  uint32_t* tagbits;    // [B][3] tag of each repetition (bit i)
  uint32_t* chal;       // [B][3]
  uint32_t* chal_full;  // [B][8] or null: the whole SHA-256 of the exp challenge (the aggregate's weights)
  uint8_t* gk_ok_len;   // [B] 1 if the GK length check passes (gk.ts:208-218)
  uint8_t* gk_tape_bad; // [B] or null: a GK draw was out of range — recorded here and folded into status[] by VReduceTask when
                        //     the GK chain runs beside the exp chain (same precedence as running it after), else written at once
  uint32_t* r_aff;      // [B][16]
  uint32_t* q_aff;      // [B][16]
  uint8_t* q_inf;       // [B]
  uint32_t* rpows;      // [B][RT_NWIN][24]
  uint32_t* rrows;      // [B][RT_NWIN][RT_ROW][24]
  uint32_t* rtab;       // [B][RT_NWIN][RT_ROW][16]
  uint32_t* samp_idx;   // [B][20] sampled repetition index
  uint32_t* samp_draw;  // [B][20] first exp draw of the sample (32-byte units from the exp area)
  // per sample (B*20)
  uint32_t* sp_T;       // [B*20][24] projective T or T1
  uint32_t* sp_T_aff;   // [B*20][16]
  uint8_t* sp_T_inf;    // [B*20]
  // per sample: 2 fixed-base jobs (T1x, T1y) and 5 derived points
  uint32_t *ta_jv, *ta_jr, *ta_proj, *ta_aff;   // [B*20*2]
  uint32_t *td_proj, *td_aff;                   // [B*20*5]
  uint8_t* td_bytes;
  uint32_t* item_chal;  // [B*20][6][3]
  // MSM entries
  uint32_t* ent_scalar; // [B][V_ENT_TOM][8]   canonical mod q
  uint32_t* ent_off;    // [B][V_ENT_TOM]      byte offset of the point inside the proof
  uint32_t* ent_pre;    // [B][V_ENT_TOM][32]  parsed TomPre
  uint32_t* ent_cnt;    // [B][20]             entries used by sample j (2 or 34)
  uint32_t* part;       // [B*20][56]          partial sums (Montgomery mod q / mod n)
  uint32_t* nent_scalar;// [B][21][8]          canonical mod n
  uint32_t* nent_aff;   // [B][21][16]
  uint8_t* nent_skip;   // [B][21]
  // GK
  uint32_t* gk_scalar;  // [B][4n+1][8]        row b: cl ca cb cd com in its first 4 n_row(b) + 1, zero scalars behind them
  uint32_t* gk_part;    // [B][2^(n-k)][8] block sums of the ring polynomial (only when n > GK_BLOCK_BITS)
  uint32_t* gk_pre;     // [B][4n+1][32]
  // fixed-base parts: tom jobs [B][2] (0: GK, 1: W) and their points; P-256 fixed part
  uint32_t *fx_jv, *fx_jr, *fx_proj;   // [B*2]
  uint32_t* nfix;       // [B][24] projective sR*R + shN*h
  uint32_t* nfix_k;     // [B][2][8] or null: sR, shN of nfix (canonical mod n) for the aggregate's weighted copy
  // MSM window sums and verdicts
  uint32_t* win_w;      // [B][MSM_NWIN][36]
  uint32_t* win_g;      // [B][MSM_NWIN][36]
  uint32_t* win_n;      // [B][MSM_NWIN_N][24]
  uint8_t* id_flags;    // [B][3]  gk, W, N identity
  int32_t* vkey;        // [B] smallest exp-side status key (vkey()), VK_NONE if none
  const uint32_t* agg_ctl;  // aggregate verdicts of the chunk (AGG_*), or null
  // outputs
  uint8_t* ok;          // [B]
  int32_t* status;      // [B]

  ZK_HD int ent_tom() const { return K * V_ENT_PER_SAMPLE + 2; }   // variable tomEdwards256 points per proof (+ keyXcom, keyYcom)
  ZK_HD int ent_nist() const { return K + 1; }                     // A_j + comS1
  ZK_HD int segs() const { return (K + V_SEG - 1) / V_SEG; }
  ZK_HD const uint8_t* proof_of(int b) const { return proofs + (size_t)b * proof_stride; }
  ZK_HD const uint8_t* tape_of(int b) const { return tape + (size_t)b * tape_stride; }
  ZK_HD const uint32_t* ring_of_row(int b) const { return ring_of ? ring_m + (size_t)8 * ring_base[ring_of[b]] : ring_m; }
  ZK_HD int n_row(int b) const { return ring_of ? (int)ring_depth[ring_of[b]] : n; }   // the depth of row b's ring
  // a row's tape has the layout of its own ring: 2 n_row(b) + 1 GK drains, the index area, the exp drains
  ZK_HD size_t gk_tape_bytes(int b) const { return mode == 1 ? 0 : (size_t)32 * (2 * n_row(b) + 1); }
  ZK_HD const uint8_t* exp_tape(int b) const { return tape_of(b) + gk_tape_bytes(b) + V_IDX_PAD; }
  ZK_HD size_t ta_pt(size_t sample, int j) const { return sample * 2 + j; }   // 0 T1x, 1 T1y
  ZK_HD size_t td_pt(size_t sample, int j) const { return sample * DERS_PER_ITEM + j; }
};

// ---------------------------------------------------------------------------------------------
// V1 — layout, statement (zkpAttestList.ts:153-164) and R/Q.  One thread per proof.
// ---------------------------------------------------------------------------------------------
struct VLayoutTask {
  VerifyCtx c;
  ZK_HD void operator()(int b) const {
    using Fn = P256n;
    using Fp = P256p;
    c.status[b] = ZKA_OK;
    c.vkey[b] = VK_NONE;
    c.ok[b] = 0;
    const uint8_t* pr = c.proof_of(b);
    const uint32_t len = c.proof_len[b];
    bool bad = len < HEAD_LEN || len > c.proof_stride;
    uint32_t off = HEAD_LEN, tg[3] = {0, 0, 0};
    for (int i = 0; i < c.S && !bad; i++) {
      if (off + 1 > len) { bad = true; break; }
      const uint8_t tag = pr[off];
      if (tag > 1) { bad = true; break; }
      c.rep_off[(size_t)b * c.S + i] = off;
      if (tag) tg[i >> 5] |= 1u << (i & 31);
      off += tag ? REP1_LEN : REP0_LEN;
      if (off > len) bad = true;
    }
    int ngk = 0;
    if (!bad && c.mode == 1) {           // verifyExp alone: the row ends with the last repetition
      if (off != len) bad = true;
      uint32_t z[8];
      zero_n<8>(z);                      // no GK instance: its fixed-base job is 0*g + 0*h
      st<8>(c.fx_jv + (size_t)b * 2 * 8, z);
      st<8>(c.fx_jr + (size_t)b * 2 * 8, z);
    } else if (!bad) {
      if (off + 1 > len) bad = true;
      else {
        ngk = pr[off];
        if (off + (uint32_t)gk_len(ngk) != len) bad = true;
      }
    }
    st<3>(c.tagbits + (size_t)b * 3, tg);
    c.gk_off[b] = off;
    c.gk_ok_len[b] = (!bad && (c.mode == 1 || ngk == c.n_row(b))) ? 1 : 0;
    if (bad) {
      ZK_SET_STATUS(c.status + b, ZKA_ERR_MALFORMED);
      // park the offsets on the header so later stages read in-bounds garbage
      for (int i = 0; i < c.S; i++) c.rep_off[(size_t)b * c.S + i] = 0;
      c.gk_off[b] = 0;
    }
    // R, rinv, z1, Q
    P256Aff R;
    bool rinf = false;
    bool okR = bad ? true : p256_parse(R, rinf, pr);
    if (bad) p256_set_generator(R);
    if (!okR) { ZK_SET_STATUS(c.status + b, ZKA_ERR_MALFORMED); p256_set_generator(R); }
    // R at infinity is reported by VChallengeTask, behind every deserialisation error of the proof
    p256_st_aff(c.r_aff + (size_t)b * 16, R);
    if (c.mode == 1) {   // Q is an input (or absent): no statement to derive it from
      P256Aff Qa;
      bool qinf = true, okq = true;
      if (c.q_ext) okq = p256_parse(Qa, qinf, c.q_ext + (size_t)b * NP);
      if (!okq) ZK_SET_STATUS(c.status + b, ZKA_ERR_MALFORMED);
      if (qinf || !okq) p256_set_generator(Qa);
      p256_st_aff(c.q_aff + (size_t)b * 16, Qa);
      c.q_inf[b] = (qinf || !okq) ? 1 : 0;
      return;
    }
    uint32_t z[8], rx[8], zm[8], rm[8], rinv[8], t[8], z1[8];
    limbs_from_be<8>(z, c.msg_hash + (size_t)b * 32, 32);
    reduce_once<FnP256>(z);
    Fp::from_mont(rx, R.x);          // coordR.x as an integer (:161), reduced mod n
    reduce_once<FnP256>(rx);
    Fn::to_mont(zm, z);
    Fn::to_mont(rm, rx);
    Fn::inv(rinv, rm);
    Fn::mul(t, rinv, zm);
    Fn::from_mont(z1, t);
    P256Pt Q;
    p256_set_identity(Q);
    p256_accum_fixed(Q, c.g_tab8, z1, 8);
    P256Aff Qa;
    const bool qinf = p256_is_identity(Q);
    if (qinf) {
      p256_set_generator(Qa);
    } else {
      uint32_t zi[8];
      Fp::inv(zi, Q.z);
      Fp::mul(Qa.x, Q.x, zi);
      Fp::mul(Qa.y, Q.y, zi);
    }
    p256_st_aff(c.q_aff + (size_t)b * 16, Qa);
    c.q_inf[b] = qinf ? 1 : 0;
  }
};

// ---------------------------------------------------------------------------------------------
// V2 — full deserialisation checks (what readJson/deserializePoint/deserializeScalar would
// reject: weier.ts:74-89, edwards.ts:70-86, group.ts:62-66).  One thread per (proof, slot):
// slot < S validates repetition `slot`, slot == S the header + GK block.
// ---------------------------------------------------------------------------------------------
struct VValidateTask {
  VerifyCtx c;
  // (one thread per (proof, slot, part-of-repetition) was slower — more threads re-reading
  //  the same headers; kept at one thread per (proof, slot))
  ZK_HD void operator()(int t) const {
    const int S1 = c.S + 1;
    const int b = t / S1, slot = t % S1;
    if (c.status[b] == ZKA_ERR_MALFORMED) return;
    const uint8_t* pr = c.proof_of(b);
    bool ok = true;
    uint32_t r[8];
    P256Aff a;
    bool inf;
    if (slot == c.S) {
      ok = p256_parse(a, inf, pr + NP) && ok;             // comS1 (R is checked in VLayoutTask)
      ok = valid_points(pr + 2 * NP, 2) && ok;            // keyXcom keyYcom
      if (c.mode != 1) {
        const uint8_t* g = pr + c.gk_off[b];
        ok = valid_gk(g, g[0]) && ok;
      }
    } else {
      const uint8_t* rep = pr + c.rep_off[(size_t)b * c.S + slot];
      ok = p256_parse(a, inf, rep + 1) && ok;
      ok = valid_points(rep + 1 + NP, 2) && ok;
      const uint8_t* body = rep + REP_HEAD;
      ok = nscalar_parse(r, body) && ok;
      ok = nscalar_parse(r, body + NS) && ok;
      if (rep[0]) {
        ok = valid_scalars(body + 2 * NS, 2) && ok;
      } else {
        const uint8_t* pa = body + 2 * NS;
        ok = valid_point_add(pa) && ok;
        ok = valid_scalars(pa + PA_LEN, 2) && ok;
      }
    }
    if (!ok) ZK_SET_STATUS(c.status + b, ZKA_ERR_MALFORMED);
  }
};

// ---------------------------------------------------------------------------------------------
// V3 — exp challenge (exp.ts:253-259), generateIndices (exp.ts:95-109) and the packed draw
// offsets of the sampled repetitions.  One thread per proof.
// ---------------------------------------------------------------------------------------------
struct VChallengeTask {
  VerifyCtx c;
  ZK_HD void operator()(int b) const {
    const uint8_t* pr = c.proof_of(b);
    // 'R is at infinity' (zkpAttestList.ts:158-160) is thrown once the whole proof has parsed (readJson): after
    // VValidateTask, so that a proof with both reports ZKA_ERR_MALFORMED.  The identity is the all-zero slot (p256_parse).
    bool rinf = true;
    for (int k = 0; k < NP; k++) rinf = rinf && pr[k] == 0;
    if (rinf) ZK_SET_STATUS(c.status + b, ZKA_ERR_R_INFINITY);
    Sha256 h;
    h.init();
    h.update(pr + 2 * NP, 2 * WP);
    for (int i = 0; i < c.S; i++) h.update(pr + c.rep_off[(size_t)b * c.S + i] + 1, NP + 2 * WP);
    uint32_t c3[3];
    h.final80(c3);
    st<3>(c.chal + (size_t)b * 3, c3);
    if (c.chal_full) st<8>(c.chal_full + (size_t)b * 8, h.h);
    // Knuth shuffle with the pre-filtered index bytes: j = rnd(limit - i) + i
    uint8_t perm[MAX_REPS];
    for (int i = 0; i < c.S; i++) perm[i] = (uint8_t)i;
    const uint8_t* ib = c.tape_of(b) + c.gk_tape_bytes(b);
    int key = VK_NONE;
    for (int i = 0; i < c.S - 2; i++) {
      uint32_t r = ib[i];
      if (r >= (uint32_t)(c.S - i)) { key = vkey(-1, 0, ZKA_ERR_TAPE_RANGE); r = 0; }
      const int j = (int)r + i;
      const uint8_t k = perm[i];
      perm[i] = perm[j];
      perm[j] = k;
    }
    uint32_t tg[3];
    ld<3>(tg, c.tagbits + (size_t)b * 3);
    uint32_t draw = 0;
    for (int j = 0; j < c.K; j++) {
      const int i = perm[j];
      const uint32_t bit = (c3[i >> 5] >> (i & 31)) & 1u;
      const uint32_t tag = (tg[i >> 5] >> (i & 31)) & 1u;
      if (bit != tag && key == VK_NONE) key = vkey(j, VK_PARAMS, ZKA_ERR_PARAMS_NOT_FOUND);   // exp.ts:269-271,301-303
      c.samp_idx[(size_t)b * c.K + j] = (uint32_t)i;
      c.samp_draw[(size_t)b * c.K + j] = draw;
      draw += bit ? 3 : 25;
    }
    if (key != VK_NONE) ZK_POST_MIN(c.vkey + b, key);
  }
};

// V4 — T = R*alpha (bit 1) or T1 = R*z + Q (bit 0) (exp.ts:272,305,317-319). Per (proof, j).
struct VSampleP256Task {
  VerifyCtx c;
  ZK_HD void operator()(int t) const {
    const int b = t / c.K;
    const int i = c.samp_idx[t];
    const uint8_t* rep = c.proof_of(b) + c.rep_off[(size_t)b * c.S + i];
    uint32_t s[8];
    limbs_from_be<8>(s, rep + REP_HEAD, 32);   // alpha or z: first scalar of the body
    reduce_once<FnP256>(s);
    P256Pt T;
    p256_set_identity(T);
    p256_accum_rtab(T, c.rtab + (size_t)b * RT_ENTRIES * P256_AFF_WORDS, s);
    if (!rep[0] && !c.q_inf[b]) {
      P256Aff Q;
      p256_ld_aff(Q, c.q_aff + (size_t)b * 16);
      p256_madd(T, T, Q);
    }
    p256_st_proj(c.sp_T + (size_t)t * P256_PROJ_WORDS, T);
  }
};

// V5 — recomputed commitments T1x = g*sx + h*r1, T1y = g*sy + h*r2 (exp.ts:326-329) as
// fixed-base jobs.  Per (proof, j); 1-bit samples get the zero job (unused).
struct VSampleJobsTask {
  VerifyCtx c;
  ZK_HD void operator()(int t) const {
    const int b = t / c.K;
    const int i = c.samp_idx[t];
    const uint8_t* rep = c.proof_of(b) + c.rep_off[(size_t)b * c.S + i];
    uint32_t v[8], r[8];
    for (int xy = 0; xy < 2; xy++) {
      zero_n<8>(v);
      zero_n<8>(r);
      if (!rep[0]) {
        P256p::from_mont(v, c.sp_T_aff + (size_t)t * 16 + 8 * xy);
        wscalar_parse(r, rep + REP_HEAD + 2 * NS + PA_LEN + xy * WS);
      }
      st<8>(c.ta_jv + c.ta_pt(t, xy) * 8, v);
      st<8>(c.ta_jr + c.ta_pt(t, xy) * 8, r);
    }
    if (c.sp_T_inf[t]) ZK_POST_MIN(c.vkey + b, vkey(t % c.K, VK_T_INF, rep[0] ? ZKA_ERR_T_INFINITY : ZKA_ERR_T1_INFINITY));  // exp.ts:283,323
  }
};

// V6 — C7, C9, C12, Cint, Cint2 (pointAdd.ts:213-215,236,248) by point addition (point_add_derived). Per (proof, j).
struct VDerivedTask {
  VerifyCtx c;
  ZK_HD void frombytes(TomPt& p, const uint8_t* b) const {
    uint32_t x[PGL], y[PGL];
    tom_parse(x, y, b);
    tom_from_affine(p, x, y);
  }
  ZK_HD void operator()(int t) const {
    const int b = t / c.K;
    const int i = c.samp_idx[t];
    const uint8_t* pr = c.proof_of(b);
    const uint8_t* rep = pr + c.rep_off[(size_t)b * c.S + i];
    TomPt pkX, pkY, Tx, Ty, T1x, T1y;
    frombytes(pkX, pr + 2 * NP);
    frombytes(pkY, pr + 2 * NP + WP);
    frombytes(Tx, rep + 1 + NP);
    frombytes(Ty, rep + 1 + NP + WP);
    uint32_t x[PGL], y[PGL];
    ld<PGL>(x, c.ta_aff + c.ta_pt(t, 0) * TOM_AFF_WORDS); ld<PGL>(y, c.ta_aff + c.ta_pt(t, 0) * TOM_AFF_WORDS + PGL);
    tom_from_affine(T1x, x, y);
    ld<PGL>(x, c.ta_aff + c.ta_pt(t, 1) * TOM_AFF_WORDS); ld<PGL>(y, c.ta_aff + c.ta_pt(t, 1) * TOM_AFF_WORDS + PGL);
    tom_from_affine(T1y, x, y);
    point_add_derived(DerivedProj{c.td_proj, c.td_pt(t, 0)}, T1x, pkX, Tx, T1y, pkY, Ty);   // exp.ts:331-341
  }
};

// V7 — the six challenges of a sampled 0-bit repetition (mult.ts:156, equality.ts:101), h in HASHES_PER_ITEM order.
// One thread per (proof, j, h).
struct VItemHashTask {
  VerifyCtx c;
  ZK_HD void operator()(int t) const {
    const int sample = t / HASHES_PER_ITEM, h = t % HASHES_PER_ITEM;
    const int b = sample / c.K;
    const int i = c.samp_idx[sample];
    const uint8_t* rep = c.proof_of(b) + c.rep_off[(size_t)b * c.S + i];
    uint32_t c3[3] = {0, 0, 0};
    if (!rep[0]) pa_challenge(c3, h, c.td_bytes + c.td_pt(sample, 0) * BSTRIDE, c.tg_bytes, rep + REP_HEAD + 2 * NS);
    st<3>(c.item_chal + (size_t)t * 3, c3);
  }
};

// ---------------------------------------------------------------------------------------------
// V8 — relations of one sampled repetition folded into (variable-point scalars, fixed-base
// partial sums); a 0-bit repetition's PointAddProof through fold_point_add (zk_sigma.cuh).
// All arithmetic mod q = tom.order in Montgomery form.  Per (proof, j).
// ---------------------------------------------------------------------------------------------
struct VRelationsTask {
  VerifyCtx c;
  ZK_HD void operator()(int t) const {
    using F = Tomq;
    using Fn = P256n;
    const int b = t / c.K, j = t % c.K;
    const int i = c.samp_idx[t];
    const uint8_t* pr = c.proof_of(b);
    const uint32_t roff = c.rep_off[(size_t)b * c.S + i];
    const uint8_t* rep = pr + roff;
    const uint8_t* body = rep + REP_HEAD;
    const uint8_t* dr = c.exp_tape(b) + (size_t)32 * c.samp_draw[t];
    uint32_t* part = c.part + (size_t)t * V_PART_WORDS;
    const Entries out{c.ent_scalar, c.ent_off};
    const size_t e0 = (size_t)b * c.ent_tom() + (size_t)j * V_ENT_PER_SAMPLE;   // Tx, Ty, then the PointAddProof's points
    SigmaFold f;
    uint32_t pX[8], pY[8], sR[8], sH[8], sC[8];
    zero_n<8>(f.gW); zero_n<8>(f.hW); zero_n<8>(pX); zero_n<8>(pY); zero_n<8>(sR); zero_n<8>(sH); zero_n<8>(sC);
    f.tape_ok = true;
    // --- multiN: relA (exp.ts:273-279 / 306-316)
    uint32_t rho[8], rm[8], s[8], sm[8], t0[8], t1[8];
    const bool first_ok = vdraw(rho, dr, true);
    Fn::to_mont(rm, rho);
    nscalar_parse(s, body);            // alpha | z
    Fn::to_mont(sm, s);
    Fn::mul(sR, rm, sm);               // rho * alpha  (coefficient of R, T = alpha R)
    nscalar_parse(s, body + NS);       // beta1 | z2
    Fn::to_mont(sm, s);
    Fn::mul(sH, rm, sm);
    if (!rep[0]) copy_n<8>(sC, rm);    // + rho * comS1
    {
      uint32_t neg[8], z[8];
      zero_n<8>(z);
      Fn::sub(neg, z, rho);            // -rho mod n, canonical
      st<8>(c.nent_scalar + ((size_t)b * c.ent_nist() + j) * 8, neg);
    }
    // coordinates of T / T1 as proof-group scalars
    uint32_t sx[8], sy[8];
    const uint32_t offTx = roff + 1 + NP, offTy = offTx + WP;
    if (rep[0]) {
      // relTx, relTy (exp.ts:284-298): sx g + beta2 h - Tx ; sy g + beta3 h - Ty
      uint32_t b2[8], b3[8], neg[8], z[8];
      ld<8>(sx, c.sp_T_aff + (size_t)t * 16);
      ld<8>(sy, c.sp_T_aff + (size_t)t * 16 + 8);
      zero_n<8>(z);
      wscalar_parse(b2, body + 2 * NS);
      wscalar_parse(b3, body + 2 * NS + WS);
      f.tape_ok = vdraw(rho, dr + 32, false) && f.tape_ok;
      F::to_mont(rm, rho);
      F::mul(t0, rm, sx); F::add(f.gW, f.gW, t0);
      F::to_mont(t1, b2); F::mul(t0, rm, t1); F::add(f.hW, f.hW, t0);
      F::sub(neg, z, rm); out.put_m(e0 + 0, neg, offTx);
      f.tape_ok = vdraw(rho, dr + 64, false) && f.tape_ok;
      F::to_mont(rm, rho);
      F::mul(t0, rm, sy); F::add(f.gW, f.gW, t0);
      F::to_mont(t1, b3); F::mul(t0, rm, t1); F::add(f.hW, f.hW, t0);
      F::sub(neg, z, rm); out.put_m(e0 + 1, neg, offTy);
      c.ent_cnt[t] = 2;
    } else {
      // aggregatePointAdd(T1x, T1y, pkX, pkY, Tx, Ty) (exp.ts:331-341): C1..C6 = T1x pkX Tx T1y pkY Ty
      const uint8_t* pa = body + 2 * NS;
      uint32_t a[PA_NCOM][8], in[6][8], r1[8], r2[8];
      fold_point_add(f, a, c.item_chal + (size_t)t * HASHES_PER_ITEM * 3, pa, dr + 32, out, e0 + 2, roff + REP_HEAD + 2 * NS);
      point_add_expand(in, a);
      // C1 = T1x = sx g + r1 h, C4 = T1y = sy g + r2 h (exp.ts:326-329) are folded onto g and h
      ld<8>(sx, c.sp_T_aff + (size_t)t * 16);
      ld<8>(sy, c.sp_T_aff + (size_t)t * 16 + 8);
      wscalar_parse(r1, pa + PA_LEN); F::to_mont(r1, r1);
      wscalar_parse(r2, pa + PA_LEN + WS); F::to_mont(r2, r2);
      F::mul(t0, in[0], sx); F::add(f.gW, f.gW, t0);
      F::mul(t0, in[0], r1); F::add(f.hW, f.hW, t0);
      F::mul(t0, in[3], sy); F::add(f.gW, f.gW, t0);
      F::mul(t0, in[3], r2); F::add(f.hW, f.hW, t0);
      copy_n<8>(pX, in[1]);
      copy_n<8>(pY, in[4]);
      out.put_m(e0 + 0, in[2], offTx);
      out.put_m(e0 + 1, in[5], offTy);
      c.ent_cnt[t] = V_ENT_PER_SAMPLE;
    }
    if (!first_ok || !f.tape_ok) ZK_POST_MIN(c.vkey + b, vkey(j, first_ok ? VK_DRAWS : VK_FIRST_DRAW, ZKA_ERR_TAPE_RANGE));
    st<8>(part, f.gW); st<8>(part + 8, f.hW); st<8>(part + 16, pX); st<8>(part + 24, pY);
    st<8>(part + 32, sR); st<8>(part + 40, sH); st<8>(part + 48, sC);
    // multiN variable point A_i
    P256Aff A;
    bool inf;
    p256_parse(A, inf, rep + 1);
    p256_st_aff(c.nent_aff + ((size_t)b * c.ent_nist() + j) * 16, A);
    c.nent_skip[(size_t)b * c.ent_nist() + j] = inf ? 1 : 0;
  }
};

// V9 — per proof: fold the 20 partial sums, emit the fixed-base jobs and the keyXcom/keyYcom/
// comS1 entries; evaluate sR*R + shN*h_nist.  One thread per proof.
struct VReduceTask {
  VerifyCtx c;
  ZK_HD void operator()(int b) const {
    using F = Tomq;
    using Fn = P256n;
    if (c.gk_tape_bad && c.gk_tape_bad[b]) ZK_SET_STATUS(c.status + b, ZKA_ERR_TAPE_RANGE);   // behind MALFORMED, R at infinity
    uint32_t gW[8], hW[8], pX[8], pY[8], sR[8], sH[8], sC[8];
    zero_n<8>(gW); zero_n<8>(hW); zero_n<8>(pX); zero_n<8>(pY); zero_n<8>(sR); zero_n<8>(sH); zero_n<8>(sC);
    for (int j = 0; j < c.K; j++) {
      const uint32_t* p = c.part + ((size_t)b * c.K + j) * V_PART_WORDS;
      uint32_t t[8];
      ld<8>(t, p); F::add(gW, gW, t);
      ld<8>(t, p + 8); F::add(hW, hW, t);
      ld<8>(t, p + 16); F::add(pX, pX, t);
      ld<8>(t, p + 24); F::add(pY, pY, t);
      ld<8>(t, p + 32); Fn::add(sR, sR, t);
      ld<8>(t, p + 40); Fn::add(sH, sH, t);
      ld<8>(t, p + 48); Fn::add(sC, sC, t);
    }
    uint32_t v[8];
    // fixed-base job 1 (W): gW g + hW h
    F::from_mont(v, gW); st<8>(c.fx_jv + ((size_t)b * 2 + 1) * 8, v);
    F::from_mont(v, hW); st<8>(c.fx_jr + ((size_t)b * 2 + 1) * 8, v);
    // keyXcom / keyYcom entries
    size_t idx = (size_t)b * c.ent_tom() + (size_t)c.K * V_ENT_PER_SAMPLE;
    F::from_mont(v, pX); st<8>(c.ent_scalar + idx * 8, v); c.ent_off[idx] = 2 * NP;
    F::from_mont(v, pY); st<8>(c.ent_scalar + (idx + 1) * 8, v); c.ent_off[idx + 1] = 2 * NP + WP;
    // multiN: comS1 entry and the fixed part
    Fn::from_mont(v, sC);
    st<8>(c.nent_scalar + ((size_t)b * c.ent_nist() + c.K) * 8, v);
    P256Aff cs;
    bool inf;
    p256_parse(cs, inf, c.proof_of(b) + NP);
    p256_st_aff(c.nent_aff + ((size_t)b * c.ent_nist() + c.K) * 16, cs);
    c.nent_skip[(size_t)b * c.ent_nist() + c.K] = inf ? 1 : 0;
    uint32_t kR[8], kH[8];
    Fn::from_mont(kR, sR);
    Fn::from_mont(kH, sH);
    P256Pt acc;
    p256_set_identity(acc);
    p256_accum_rtab(acc, c.rtab + (size_t)b * RT_ENTRIES * P256_AFF_WORDS, kR);
    p256_accum_fixed(acc, c.h_tab8, kH, c.h_w);
    p256_st_proj(c.nfix + (size_t)b * P256_PROJ_WORDS, acc);
    if (c.nfix_k) {   // for the aggregate's weighted copy (AggNistFixWeightTask); the per-proof path reads nfix
      st<8>(c.nfix_k + (size_t)b * 16, kR);
      st<8>(c.nfix_k + (size_t)b * 16 + 8, kH);
    }
  }
};

// V10 — parse the variable tomEdwards256 points of the MSMs into table-entry form.
struct VParseEntriesTask {
  const uint8_t* proofs;
  size_t proof_stride;
  const uint32_t* off;   // [count] byte offset inside the proof
  uint32_t* pre;         // [count][32]
  int per_proof;
  ZK_HD void operator()(int t) const {
    const int b = t / per_proof;
#if defined(ZKA_PG_WAR256)
    uint32_t x[8], y[8];
    tom_parse(x, y, proofs + (size_t)b * proof_stride + off[t]);
    uint32_t* o = pre + (size_t)t * TOM_PRE_WORDS;
    st<8>(o, x); st<8>(o + 8, y);
#else
    using F = Tomp;
    uint32_t x[9], y[9], k[9], d1[9];
    tom_parse(x, y, proofs + (size_t)b * proof_stride + off[t]);
    tom_const(d1, TOM_D1);
    F::mul(k, x, y);
    F::mul(k, k, d1);
    F::reduce(x); F::reduce(y); F::reduce(k);
    uint32_t* o = pre + (size_t)t * TOM_PRE_WORDS;
    st<9>(o, x); st<9>(o + 9, y); st<9>(o + 18, k);
#endif
  }
};

// V11a — large rings only (n > GK_BLOCK_BITS): the N*n multiplications of the ring polynomial, one
// thread per (proof, block of 2^GK_BLOCK_BITS ring entries).  Every thread re-derives the challenge
// x = H(cl, ca, cb, cd) and the f_j from the proof (cheap next to its 3 * 1024 multiplications).
struct VGkSumTask {
  VerifyCtx c;
  ZK_HD void operator()(int t) const {
    using F = Tomq;
    const int gblk = 1 << (c.n - gk_block_bits(c.n));   // the grid: gblk blocks per proof
    const int b = t / gblk, blk = t % gblk;
    const int n = c.n_row(b), k = gk_block_bits(n);
    if (n == k || blk >= 1 << (n - k)) return;   // VGkTask sums a ring of one block itself
    uint32_t acc[8];
    zero_n<8>(acc);
    if (c.gk_ok_len[b]) {
      const uint8_t* g = c.proof_of(b) + c.gk_off[b];
      const uint8_t* pts = g + 1;
      const uint8_t* fs = pts + (size_t)4 * n * WP;
      Sha256 h;
      h.init();
      h.update(pts, 4 * n * WP);
      uint32_t c3[3], xc[8], xm[8];
      h.final80(c3);
      challenge_to_limbs(xc, c3);
      F::to_mont(xm, xc);
      uint32_t fm[20][8], omf[20][8];
      for (int i = 0; i < n; i++) {
        uint32_t f[8];
        wscalar_parse(f, fs + (size_t)i * WS);
        F::to_mont(fm[i], f);
        F::sub(omf[i], xm, fm[i]);
      }
      gk_block_sum(acc, c.ring_of_row(b), omf, fm, n, k, (uint32_t)blk, nullptr);
    }
    st<8>(c.gk_part + (size_t)t * 8, acc);
  }
};

// ---------------------------------------------------------------------------------------------
// V11 — Groth-Kohlweiss relations (gk.ts:220-259).  One thread per proof.
// ---------------------------------------------------------------------------------------------
struct VGkTask {
  VerifyCtx c;
  ZK_HD void operator()(int b) const {
    using F = Tomq;
    const int n = c.n_row(b), per = 4 * c.n + 1;
    if (c.gk_tape_bad) c.gk_tape_bad[b] = 0;
    // the slots behind the row's 4n + 1 entries (all of them when the length check fails) hold zero scalars
    for (int k = c.gk_ok_len[b] ? 4 * n + 1 : 0; k < per; k++) { uint32_t z[8]; zero_n<8>(z); st<8>(c.gk_scalar + ((size_t)b * per + k) * 8, z); }
    if (!c.gk_ok_len[b]) {   // length check fails -> verifyMembership returns false before any draw
      uint32_t z[8]; zero_n<8>(z);
      st<8>(c.fx_jv + (size_t)b * 2 * 8, z); st<8>(c.fx_jr + (size_t)b * 2 * 8, z);
      return;
    }
    const uint8_t* g = c.proof_of(b) + c.gk_off[b];
    const uint8_t* pts = g + 1;
    const uint8_t* fs = pts + (size_t)4 * n * WP;
    const uint8_t* zas = fs + (size_t)n * WS;
    const uint8_t* zbs = zas + (size_t)n * WS;
    const uint8_t* zds = zbs + (size_t)n * WS;
    Sha256 h;
    h.init();
    h.update(pts, 4 * n * WP);
    uint32_t c3[3], xc[8], xm[8];
    h.final80(c3);
    challenge_to_limbs(xc, c3);
    F::to_mont(xm, xc);
    const uint8_t* dr = c.tape_of(b);
    uint32_t gS[8], hS[8], t0[8], t1[8], rho[8], r0[8], r1[8], z[8];
    zero_n<8>(gS); zero_n<8>(hS); zero_n<8>(z);
    uint32_t fm[20][8], omf[20][8];     // f_j and x - f_j (Montgomery)
    bool tape_ok = true;
    uint32_t* sc = c.gk_scalar + (size_t)b * per * 8;
    for (int i = 0; i < n; i++) {
      uint32_t f[8], za[8], zb[8];
      wscalar_parse(f, fs + (size_t)i * WS);  F::to_mont(fm[i], f);
      wscalar_parse(za, zas + (size_t)i * WS); F::to_mont(za, za);
      wscalar_parse(zb, zbs + (size_t)i * WS); F::to_mont(zb, zb);
      F::sub(omf[i], xm, fm[i]);
      tape_ok = vdraw(rho, dr + 32 * (2 * i), false) && tape_ok;     F::to_mont(r0, rho);
      tape_ok = vdraw(rho, dr + 32 * (2 * i + 1), false) && tape_ok; F::to_mont(r1, rho);
      // rel0: x cl + ca - f g - za h ; rel1: (x - f) cl + cb - zb h
      F::mul(t0, r0, xm); F::mul(t1, r1, omf[i]); F::add(t0, t0, t1);
      F::from_mont(t1, t0); st<8>(sc + (size_t)i * 8, t1);                 // cl_i
      F::from_mont(t1, r0); st<8>(sc + (size_t)(n + i) * 8, t1);           // ca_i
      F::from_mont(t1, r1); st<8>(sc + (size_t)(2 * n + i) * 8, t1);       // cb_i
      F::mul(t0, r0, fm[i]); F::sub(gS, gS, t0);
      F::mul(t0, r0, za); F::sub(hS, hS, t0);
      F::mul(t0, r1, zb); F::sub(hS, hS, t0);
    }
    // total = sum_i v_i prod_j (bit_j(i) ? f_j : x - f_j)   (gk.ts:239-250)
    uint32_t total[8];
    {
      const int k = gk_block_bits(n), nblk = 1 << (n - k);
      if (nblk == 1) {
        gk_block_sum(total, c.ring_of_row(b), omf, fm, n, k, 0u, nullptr);
      } else {               // block sums from VGkSumTask
        uint32_t v[8];
        zero_n<8>(total);
        for (int i = 0; i < nblk; i++) {
          ld<8>(v, c.gk_part + ((size_t)b * (1 << (c.n - gk_block_bits(c.n))) + i) * 8);
          F::add(total, total, v);
        }
      }
    }
    // relFinal: sum_k -x^k cd_k + x^n com - total g - zd h
    uint32_t rf[8], xp[8], zd[8];
    tape_ok = vdraw(rho, dr + 32 * (2 * n), false) && tape_ok;
    F::to_mont(rf, rho);
    F::set_one(xp);
    for (int k = 0; k < n; k++) {
      F::mul(t0, rf, xp);
      F::sub(t0, z, t0);
      F::from_mont(t1, t0); st<8>(sc + (size_t)(3 * n + k) * 8, t1);       // cd_k
      F::mul(xp, xp, xm);
    }
    F::mul(t0, rf, xp);
    F::from_mont(t1, t0); st<8>(sc + (size_t)(4 * n) * 8, t1);             // com = keyXcom
    F::mul(t0, rf, total); F::sub(gS, gS, t0);
    wscalar_parse(zd, zds); F::to_mont(zd, zd);
    F::mul(t0, rf, zd); F::sub(hS, hS, t0);
    F::from_mont(t1, gS); st<8>(c.fx_jv + (size_t)b * 2 * 8, t1);
    F::from_mont(t1, hS); st<8>(c.fx_jr + (size_t)b * 2 * 8, t1);
    if (!tape_ok) {
      if (c.gk_tape_bad) c.gk_tape_bad[b] = 1;
      else ZK_SET_STATUS(c.status + b, ZKA_ERR_TAPE_RANGE);
    }
  }
};
struct VGkOffsetsTask {   // byte offsets of cl, ca, cb, cd, com for VParseEntriesTask
  VerifyCtx c;
  uint32_t* off;          // [B][4n+1]
  ZK_HD void operator()(int t) const {
    const int per = 4 * c.n + 1;
    const int b = t / per, k = t % per;   // com and the zero-scalar slots behind it read keyXcom
    off[t] = c.gk_ok_len[b] && k < 4 * c.n_row(b) ? c.gk_off[b] + 1 + (uint32_t)k * WP : (uint32_t)(2 * NP);
  }
};

// ---------------------------------------------------------------------------------------------
// Bucket MSM over tomEdwards256 (replaces MultiMult.evaluate, multimult.ts:61-89).
// One thread per (instance, window): 2^c - 1 buckets in local memory, mixed additions into
// buckets, then the running-sum reduction.  Instances: GK (4n+1 entries) and multiW.
// ---------------------------------------------------------------------------------------------
struct alignas(16) U4 { uint32_t x, y, z, w; };
#if defined(ZKA_PG_WAR256)
enum : int { PG_EXT_WORDS = 24, PG_EXT_U4 = 6 };   // a parked projective point: X, Y, Z
ZK_HD void bk_load(TomPt& p, const U4* b) {
  uint32_t w[24];
#pragma unroll
  for (int i = 0; i < 6; i++) { const U4 u = b[i]; w[4 * i] = u.x; w[4 * i + 1] = u.y; w[4 * i + 2] = u.z; w[4 * i + 3] = u.w; }
#pragma unroll
  for (int i = 0; i < 8; i++) { p.x[i] = w[i]; p.y[i] = w[8 + i]; p.z[i] = w[16 + i]; }
}
ZK_HD void bk_store(U4* b, const TomPt& p) {
  uint32_t w[24];
#pragma unroll
  for (int i = 0; i < 8; i++) { w[i] = p.x[i]; w[8 + i] = p.y[i]; w[16 + i] = p.z[i]; }
#pragma unroll
  for (int i = 0; i < 6; i++) { U4 u; u.x = w[4 * i]; u.y = w[4 * i + 1]; u.z = w[4 * i + 2]; u.w = w[4 * i + 3]; b[i] = u; }
}
#else
enum : int { PG_EXT_WORDS = 36, PG_EXT_U4 = 9 };   // a parked extended point: X, Y, T, Z
ZK_HD void bk_load(TomPt& p, const U4* b) {
  uint32_t w[36];
#pragma unroll
  for (int i = 0; i < 9; i++) { const U4 u = b[i]; w[4 * i] = u.x; w[4 * i + 1] = u.y; w[4 * i + 2] = u.z; w[4 * i + 3] = u.w; }
#pragma unroll
  for (int i = 0; i < 9; i++) { p.x[i] = w[i]; p.y[i] = w[9 + i]; p.t[i] = w[18 + i]; p.z[i] = w[27 + i]; }
}
ZK_HD void bk_store(U4* b, const TomPt& p) {
  uint32_t w[36];
#pragma unroll
  for (int i = 0; i < 9; i++) { w[i] = p.x[i]; w[9 + i] = p.y[i]; w[18 + i] = p.t[i]; w[27 + i] = p.z[i]; }
#pragma unroll
  for (int i = 0; i < 9; i++) { U4 u; u.x = w[4 * i]; u.y = w[4 * i + 1]; u.z = w[4 * i + 2]; u.w = w[4 * i + 3]; b[i] = u; }
}
#endif
// Signed window digits without a carry chain: with OFFS = sum_j 32 * 64^j the unsigned 6-bit windows of
// k' = k + OFFS, minus 32, are digits d_j in [-32, 31] with sum_j d_j 64^j = k.  Returns |d_j| (the
// bucket, 0..32) and its sign.  Half the buckets of an unsigned 6-bit window, one window fewer per
// 6 bits than the 5-bit version: 43 x (n + 64) instead of 52 x (n + 62) point operations.
ZK_HD uint32_t msm_digit6(const uint32_t* k, int w, bool& neg) {
  constexpr uint32_t OFFS[9] = {0x20820820u, 0x08208208u, 0x82082082u, 0x20820820u, 0x08208208u,
                                0x82082082u, 0x20820820u, 0x08208208u, 0x00000002u};
  uint32_t kp[9];
  uint64_t c = 0;
#pragma unroll
  for (int i = 0; i < 9; i++) {
    c += (uint64_t)(i < 8 ? k[i] : 0u) + OFFS[i];
    kp[i] = (uint32_t)c;
    c >>= 32;
  }
  const int pos = w * MSM_C, wi = pos >> 5, sh = pos & 31;
  uint64_t v = 0;
#pragma unroll
  for (int i = 0; i < 9; i++) {     // static indexing: select the two limbs the window touches
    if (i == wi) v |= kp[i];
    if (i == wi + 1) v |= (uint64_t)kp[i] << 32;
  }
  const int d = (int)((uint32_t)(v >> sh) & 63u) - 32;
  neg = d < 0;
  return (uint32_t)(d < 0 ? -d : d);
}
struct MsmTomWindowTask {
  // Sorted-bucket Pippenger: a thread first counting-sorts the indices of its window's entries by
  // |digit| (2 bytes of local memory per entry), then walks the sorted entries in one flat loop,
  // summing each bucket in REGISTERS, and finally folds the bucket sums into the running sums
  //   run += S_d ; tot += run      =>   tot = sum_d d * S_d .
  // (The first version kept 31 extended points per thread in local memory and read-modify-wrote
  // one per addition: 4.5 KB/thread thrashed L1/L2, and the kernel was bound by DRAM reads instead of the
  // multiplier pipe.)
  const uint32_t* scalar;   // [inst][stride][8]
  const uint32_t* pre;      // [inst][stride][32]
  const uint32_t* cnt;      // [inst][groups] entries used per group (or null: all `group_len` used)
  int stride, groups, group_len, tail;   // entries of an instance = groups*group_len, then `tail` always-used ones
  int seg_groups, segs;     // the groups are walked in `segs` segments of <= seg_groups groups (one thread per segment
                            // and window: <= V_ENT_SEG entries each); the tail rides with segment 0
  uint32_t* win;            // [inst][segs][MSM_NWIN][PG_EXT_WORDS]
  ZK_HD void operator()(int t) const {
    const int is = t / MSM_NWIN, w = t % MSM_NWIN;
    const int inst = is / segs, seg = is % segs;
    constexpr int NB = 33;          // bucket 0 (skipped) .. 32
    const uint32_t* sc = scalar + (size_t)inst * stride * 8;
    const uint32_t* pp = pre + (size_t)inst * stride * TOM_PRE_WORDS;
    const int g0 = seg * seg_groups;
    int ng = groups - g0;
    if (ng > seg_groups) ng = seg_groups;
    if (ng < 0) ng = 0;
    const int tl = seg == 0 ? tail : 0;
    const int gbase = g0 * group_len;           // first entry of this segment's groups
    const int tbase = groups * group_len;       // first tail entry
    const int nloc = ng * group_len;            // local indices [0, nloc) are group entries, [nloc, nloc + tl) the tail
    uint16_t order[V_ENT_SEG];     // sign << 15 | (bucket - 1) << 10 | LOCAL entry index, sorted by bucket
    uint16_t start[NB + 1];
    for (int d = 0; d <= NB; d++) start[d] = 0;
    // pass 1: histogram of buckets
    for (int gidx = 0; gidx <= ng; gidx++) {
      const int m = gidx < ng ? (cnt ? (int)cnt[(size_t)inst * groups + g0 + gidx] : group_len) : tl;
      const int base = gidx < ng ? gbase + gidx * group_len : tbase;
      for (int e = 0; e < m; e++) {
        bool neg;
        const uint32_t bk = msm_digit6(sc + (size_t)(base + e) * 8, w, neg);
        start[bk + 1]++;
      }
    }
    for (int d = 1; d <= NB; d++) start[d] = (uint16_t)(start[d] + start[d - 1]);
    uint16_t fillp[NB];
    for (int d = 0; d < NB; d++) fillp[d] = start[d];
    // pass 2: scatter
    for (int gidx = 0; gidx <= ng; gidx++) {
      const int m = gidx < ng ? (cnt ? (int)cnt[(size_t)inst * groups + g0 + gidx] : group_len) : tl;
      const int base = gidx < ng ? gbase + gidx * group_len : tbase;
      const int lbase = gidx < ng ? gidx * group_len : nloc;
      for (int e = 0; e < m; e++) {
        bool neg;
        const uint32_t bk = msm_digit6(sc + (size_t)(base + e) * 8, w, neg);
        const uint32_t enc = bk ? (((neg ? 1u : 0u) << 15) | ((bk - 1) << 10) | (uint32_t)(lbase + e)) : (uint32_t)(lbase + e);
        order[fillp[bk]++] = (uint16_t)enc;
      }
    }
    // pass 3: ONE flat loop over the entries with a non-zero digit (the trip count is the same for
    // every window of an instance up to a few entries, so the warp does not diverge); a finished
    // bucket sum is parked in local memory exactly once
    U4 S[NB][PG_EXT_U4];
    uint64_t present = 0;
    TomPt acc;
    tom_set_identity(acc);
    int curd = NB - 1;
    const int total = start[NB], first = start[1];
    for (int q = total - 1; q >= first; q--) {
      const uint32_t oe = order[q];
      const int d = (int)((oe >> 10) & 31u) + 1;
      if (d != curd) {
        bk_store(S[curd], acc);
        present |= 1ull << curd;
        tom_set_identity(acc);
        curd = d;
      }
      TomPre pt;
      const int loc = (int)(oe & 1023u);
      tom_ld_pre(pt, pp + (size_t)(loc < nloc ? gbase + loc : tbase + (loc - nloc)) * TOM_PRE_WORDS);
      if (oe & 0x8000u) pg_pre_neg(pt);   // negative digit
      tom_madd<true, TompMsm>(acc, acc, pt);
    }
    bk_store(S[curd], acc);
    present |= 1ull << curd;
    // pass 4: running sums  tot = sum_d d * S_d
    TomPt run, tot;
    tom_set_identity(run);
    tom_set_identity(tot);
    for (int d = NB - 1; d >= 1; d--) {
      if ((present >> d) & 1ull) {
        bk_load(acc, S[d]);
        tom_add(run, run, acc);
      }
      tom_add(tot, tot, run);
    }
    bk_store(reinterpret_cast<U4*>(win + (size_t)t * PG_EXT_WORDS), tot);
  }
};
// Horner over the windows + the fixed-base part; verdict = identity?  One thread per instance.
struct MsmTomCombineTask {
  const uint32_t* win;      // [inst][segs][MSM_NWIN][36]
  const uint32_t* fixed;    // fixed-base commitment of instance i at fixed[(i*fix_stride + fix_off)*27]
  uint8_t* flag;            // verdict of instance i at flag[i*3 + flag_off]
  int fix_stride, fix_off, flag_off;
  int segs = 1;
  ZK_HD void operator()(int inst) const {
    TomPt acc, wsum;
    tom_set_identity(acc);
    for (int w = MSM_NWIN - 1; w >= 0; w--) {
      for (int k = 0; k < MSM_C; k++) tom_dbl(acc, acc);
      for (int sg = 0; sg < segs; sg++) {
        bk_load(wsum, reinterpret_cast<const U4*>(win + (((size_t)inst * segs + sg) * MSM_NWIN + w) * PG_EXT_WORDS));
        tom_add(acc, acc, wsum);
      }
    }
    TomPt f;
    const uint32_t* fp = fixed + ((size_t)inst * fix_stride + fix_off) * TOM_PROJ_WORDS;
    tom_ld_xyz(f.x, f.y, f.z, fp);
#if !defined(ZKA_PG_WAR256)
    // The commitment kernel works on the a = -1 image curve E2 and stores (W : V : Z) with
    // x' = W / (Z sqrt(-d1)), y = Z / V.  Same point in E1 extended coordinates with Z' = Z V:
    //   X = c W V,  Y = Z^2,  T = X Y / Z' = c W Z,   c = 1/sqrt(-d1).
    pg_fixed_to_msm(f);
#endif
    tom_add(acc, acc, f);
    const bool id = pg_is_identity(acc);
    flag[(size_t)inst * 3 + flag_off] = id ? 1 : 0;
  }
};

// Bucket MSM over P-256 (multiN): 21 points, 4-bit windows.  One thread per (proof, window).
// signed 4-bit digits without a carry chain (see msm_digit6): windows of k + sum_{j<64} 8 * 16^j, minus 8
ZK_HD uint32_t msm_digit4(const uint32_t* k, int w, bool& neg) {
  uint32_t kp[9];
  uint64_t c = 0;
#pragma unroll
  for (int i = 0; i < 8; i++) {
    c += (uint64_t)k[i] + 0x88888888u;
    kp[i] = (uint32_t)c;
    c >>= 32;
  }
  kp[8] = (uint32_t)c;
  uint32_t word = 0;
#pragma unroll
  for (int i = 0; i < 9; i++)
    if (i == (w >> 3)) word = kp[i];
  const int d = (int)((word >> (4 * (w & 7))) & 15u) - (w < 64 ? 8 : 0);
  neg = d < 0;
  return (uint32_t)(d < 0 ? -d : d);
}
struct MsmP256WindowTask {
  const uint32_t* scalar;   // [B][nent][8]
  const uint32_t* aff;      // [B][nent][16]
  const uint8_t* skip;      // [B][nent]
  uint32_t* win;            // [B][MSM_NWIN_N][24]
  int nent = V_SAMPLES + 1; // entries per proof: K sampled A_j + comS1
  const uint32_t* ctl = nullptr;
  ZK_HD void operator()(int t) const {
    if (ctl && ctl[AGG_NIST_PASS]) return;
    const int b = t / MSM_NWIN_N, w = t % MSM_NWIN_N;
    P256Pt bucket[8];
    for (int d = 0; d < 8; d++) p256_set_identity(bucket[d]);
    for (int e = 0; e < nent; e++) {
      if (skip[(size_t)b * nent + e]) continue;
      uint32_t k[8];
      ld<8>(k, scalar + ((size_t)b * nent + e) * 8);
      bool neg;
      const uint32_t dgt = msm_digit4(k, w, neg);
      if (dgt) {
        P256Aff q;
        p256_ld_aff(q, aff + ((size_t)b * nent + e) * 16);
        if (neg) P256p::neg(q.y, q.y);
        p256_madd(bucket[dgt - 1], bucket[dgt - 1], q);
      }
    }
    P256Pt run, tot;
    p256_set_identity(run);
    p256_set_identity(tot);
    for (int d = 7; d >= 0; d--) {
      p256_add(run, run, bucket[d]);
      p256_add(tot, tot, run);
    }
    p256_st_proj(win + (size_t)t * P256_PROJ_WORDS, tot);
  }
};
struct MsmP256CombineTask {
  const uint32_t* win;
  const uint32_t* fixed;    // [B][24]
  uint8_t* flag;            // [B][3], writes [b][2]
  ZK_HD void operator()(int b) const {
    P256Pt acc, wsum;
    p256_set_identity(acc);
    for (int w = MSM_NWIN_N - 1; w >= 0; w--) {
      for (int k = 0; k < MSM_C_N; k++) p256_dbl(acc, acc);
      p256_ld_proj(wsum, win + ((size_t)b * MSM_NWIN_N + w) * P256_PROJ_WORDS);
      p256_add(acc, acc, wsum);
    }
    P256Pt f;
    p256_ld_proj(f, fixed + (size_t)b * P256_PROJ_WORDS);
    p256_add(acc, acc, f);
    flag[(size_t)b * 3 + 2] = p256_is_identity(acc) ? 1 : 0;
  }
};

// The two tomEdwards256 MSM instances of a proof (multiW: up to 682 entries, GK: 4n+1) as one grid: the
// short GK threads fill the SMs the long multiW threads leave idle (one 1024-proof batch is 0.8 of a wave).
struct MsmTomWindowBothTask {
  MsmTomWindowTask w, gk;
  int nW, nWp;   // multiW threads (proofs x segments x windows), rounded up to a warp multiple
  int nG;        // GK threads (proofs x windows)
  const uint32_t* ctl = nullptr;
  ZK_HD void operator()(int t) const {
    if (ctl && ctl[AGG_TOM_PASS]) return;
    if (t < nWp) {
      if (t < nW) w(t);
    } else if (t - nWp < nG) {
      gk(t - nWp);
    }
  }
};

#if !defined(ZKA_HOSTSIM) && defined(ZKA_MSM_MINBLOCKS)
template <> struct TaskMinBlocks<MsmTomWindowBothTask> { static constexpr int value = ZKA_MSM_MINBLOCKS; };
#endif

// The three Horner passes of a proof (GK, multiW, multiN) are 250-doubling latency chains run by one
// thread each; launched as ONE grid they overlap instead of queueing (3 B threads are still few).
struct MsmCombineAllTask {
  MsmTomCombineTask gk, w;
  MsmP256CombineTask n;
  int B, Bp;   // Bp = B rounded up to a warp multiple: the P-256 chain never shares a warp with a Tom chain
  const uint32_t* ctl = nullptr;
  ZK_HD void operator()(int t) const {
    const int kind = t / Bp, i = t % Bp;
    if (i >= B) return;
    if (ctl && ctl[kind == 2 ? AGG_NIST_PASS : AGG_TOM_PASS]) return;
    if (kind == 0) gk(i);
    else if (kind == 1) w(i);
    else n(i);
  }
};


// ---- stand-alone sub-proof verifiers (the reference's unit-test / bench surface) -------------------------------
// Rows for the shared tasks are assembled on the device: a 264-byte header followed by the caller's proof bytes.
//   verifyExp        (exp.ts:233):  header = paramsNIST.g | Clambda | Px | Py, body = the repetitions
//   verifyMembership (gk.ts:197):   header = 0 | 0 | com | 0,              body = the GK block
struct VAssembleTask {
  const uint8_t *h0, *h1, *h2, *h3;   // [B][65] [B][65] [B][67] [B][67]; null = zero bytes
  const uint8_t* body;                // [B][body_stride]
  size_t body_stride;
  const uint32_t* body_len;           // [B]
  uint8_t* rows;                      // [B][row_stride]
  size_t row_stride;
  uint32_t* row_len;                  // [B]  = HEAD_LEN + body_len (clamped to the stride)
  int pieces;                         // 64-byte pieces per row
  ZK_HD void operator()(int t) const {
    const int b = t / pieces, j = t % pieces;
    uint32_t bl = body_len[b];
    if ((size_t)bl > body_stride) bl = (uint32_t)body_stride + 1;   // stays "too long" -> MALFORMED
    if (j == 0) row_len[b] = HEAD_LEN + bl;
    uint8_t* row = rows + (size_t)b * row_stride;
    const size_t lo = (size_t)64 * j, hi = lo + 64;
    for (size_t o = lo; o < hi && o < row_stride; o++) {
      uint8_t v = 0;
      if (o < NP) v = h0 ? h0[(size_t)b * NP + o] : 0;
      else if (o < 2 * NP) v = h1 ? h1[(size_t)b * NP + (o - NP)] : 0;
      else if (o < 2 * NP + WP) v = h2 ? h2[(size_t)b * WP + (o - 2 * NP)] : 0;
      else if (o < HEAD_LEN) v = h3 ? h3[(size_t)b * WP + (o - 2 * NP - WP)] : 0;
      else if (o - HEAD_LEN < bl && o - HEAD_LEN < body_stride) v = body[(size_t)b * body_stride + (o - HEAD_LEN)];
      row[o] = v;
    }
  }
};
// verifyMembership alone: layout + deserialisation checks of com and the GK block.  One thread per proof.
struct VGkOnlyLayoutTask {
  VerifyCtx c;
  ZK_HD void operator()(int b) const {
    c.status[b] = ZKA_OK;
    c.ok[b] = 0;
    const uint8_t* pr = c.proof_of(b);
    const uint32_t len = c.proof_len[b];
    bool bad = len < HEAD_LEN + 1 || len > c.proof_stride;
    int ngk = 0;
    if (!bad) {
      ngk = pr[HEAD_LEN];
      if (HEAD_LEN + (uint32_t)gk_len(ngk) != len) bad = true;
    }
    c.gk_off[b] = bad ? 0 : HEAD_LEN;
    bool okp = true;
    if (!bad) {
      okp = valid_points(pr + 2 * NP, 1);
      okp = valid_gk(pr + HEAD_LEN, ngk) && okp;
    }
    if (bad || !okp) ZK_SET_STATUS(c.status + b, ZKA_ERR_MALFORMED);
    c.gk_ok_len[b] = (!bad && okp && ngk == c.n) ? 1 : 0;
  }
};
struct VGkOnlyFinalTask {
  VerifyCtx c;
  ZK_HD void operator()(int b) const {
    const int st = c.status[b];
    c.ok[b] = (st == ZKA_OK && c.gk_ok_len[b] && c.id_flags[(size_t)b * 3]) ? 1 : 0;
  }
};

// ---- verifyEquality / verifyMult / verifyPointAdd alone (equality.ts:80-116, mult.ts:133-175, pointAdd.ts:181-259)
// Row = the statement's commitments (2 / 3 / 6 x 67 bytes, in the reference's argument order) followed by the proof
// (233 / 633 / 3266 bytes).  One thread per statement folds all relations under the tape's randomizers into
//   * scalars of the variable points (inputs and proof points)  -> entries of ONE Pippenger instance,
//   * the coefficients of g and h                                -> one fixed-base commitment,
// with the same folds as the batched verifier's sampled repetitions (zk_sigma.cuh); the derived commitments (C7, C9,
// C12, Cint, Cint2) are expanded onto the inputs they are sums of.
enum : int { SUB_EQ = 0, SUB_MULT = 1, SUB_PADD = 2, SUB_ENT_MAX = 6 + PA_ENTRIES };   // 38: PX..RY, PointAddProof
ZK_LAYOUT_FN int sub_points(int kind) { return kind == SUB_EQ ? 2 : kind == SUB_MULT ? 3 : 6; }
ZK_LAYOUT_FN int sub_proof_len(int kind) { return kind == SUB_EQ ? EQ_LEN : kind == SUB_MULT ? MULT_LEN : PA_LEN; }
ZK_LAYOUT_FN int sub_draws(int kind) { return kind == SUB_EQ ? 2 : kind == SUB_MULT ? 5 : 24; }
ZK_LAYOUT_FN int sub_entries(int kind) { return kind == SUB_EQ ? 4 : kind == SUB_MULT ? 9 : SUB_ENT_MAX; }

// encoding (67 bytes in a BSTRIDE slot) of an E1 affine point given as Montgomery (x', y)
#if defined(ZKA_PG_WAR256)
ZK_HD void tom_encode_affine(uint8_t* out, const uint32_t* xm, const uint32_t* ym) {
  uint32_t cx[8], cy[8];
  Warp::from_mont(cx, xm);
  Warp::from_mont(cy, ym);
  store_point_words<8, 32>(out, 0x04u, cx, cy);
}
#else
ZK_HD void tom_encode_affine(uint8_t* out, const uint32_t* x1m, const uint32_t* ym) {
  uint32_t isa[9], cx[9], cy[9];
  tom_const(isa, TOM_INVSQRTA);
  Tomp::mul(cx, x1m, isa);
  Tomp::from_mont(cx, cx);
  Tomp::from_mont(cy, ym);
  store_point_words<9, 33>(out, 0x04u, cx, cy);
}
#endif
ZK_HD void tom_encode_proj(uint8_t* out, const TomPt& p) {   // one inversion: low-volume paths only
  uint32_t zi[PGL], x[PGL], y[PGL];
  PGp::inv(zi, p.z);
  PGp::mul(x, p.x, zi);
  PGp::mul(y, p.y, zi);
  tom_encode_affine(out, x, y);
}
struct VSubProofTask {
  int kind;
  const uint8_t* rows;     // [B][stride]
  size_t stride;
  const uint8_t* tape;     // [B][tape_stride] drains (mod tom.order) in Relation.drain call order
  size_t tape_stride;
  const uint8_t* tg_bytes; // encoding of ProofGroup.g (C_14 of pi_8, pointAdd.ts:220)
  uint32_t* ent_scalar;    // [B][SUB_ENT_MAX][8] canonical
  uint32_t* ent_off;       // [B][SUB_ENT_MAX] byte offset of the point in the row
  uint32_t *fx_jv, *fx_jr; // [B][2][8]: job 1 = (coefficient of g, coefficient of h); job 0 = 0
  int32_t* status;         // [B]
  uint8_t* ok;             // [B]

  struct DerivedBytes {    // encodings of the derived points, BSTRIDE apart in DER_* order
    uint8_t* out;
    ZK_HD void operator()(int d, const TomPt& p) const { tom_encode_proj(out + (size_t)d * BSTRIDE, p); }
  };
  ZK_HD void operator()(int b) const {
    using F = Tomq;
    const uint8_t* row = rows + (size_t)b * stride;
    const uint8_t* dr = tape + (size_t)b * tape_stride;
    const int np = sub_points(kind);
    const uint8_t* proof = row + (size_t)np * WP;
    const uint32_t poff = (uint32_t)(np * WP);
    const Entries out{ent_scalar, ent_off};
    const size_t e0 = (size_t)b * SUB_ENT_MAX;
    status[b] = ZKA_OK;
    ok[b] = 0;
    // deserialisation checks of every point and scalar (deserializePoint / deserializeScalar would throw)
    bool good = valid_points(row, np);
    good = (kind == SUB_EQ ? valid_equality(proof) : kind == SUB_MULT ? valid_mult(proof) : valid_point_add(proof)) && good;
    SigmaFold f;
    zero_n<8>(f.gW); zero_n<8>(f.hW);
    f.tape_ok = true;
    uint32_t zero[8];
    zero_n<8>(zero);
    for (int e = 0; e < SUB_ENT_MAX; e++) out.put(e0 + e, zero, 0);   // unused entries: scalar 0 on the first input point
    if (!good) {
      ZK_SET_STATUS(status + b, ZKA_ERR_MALFORMED);
    } else if (kind == SUB_EQ) {
      uint32_t c3[3], a[2][8], es[2][8];
      zero_n<8>(a[0]); zero_n<8>(a[1]);
      sigma_challenge(c3, row, row + WP, nullptr, proof, 2);
      fold_equality(f, c3, proof, dr, a[0], a[1], es);
      for (int i = 0; i < 2; i++) { out.put_m(e0 + i, a[i], (uint32_t)i * WP); out.put(e0 + 2 + i, es[i], poff + (uint32_t)i * WP); }
    } else if (kind == SUB_MULT) {
      uint32_t c3[3], a[3][8], es[6][8];
      zero_n<8>(a[0]); zero_n<8>(a[1]); zero_n<8>(a[2]);
      sigma_challenge(c3, row, row + WP, row + 2 * WP, proof, 6);
      fold_mult(f, c3, proof, dr, a[0], a[1], a[2], es);
      for (int i = 0; i < 3; i++) out.put_m(e0 + i, a[i], (uint32_t)i * WP);
      for (int i = 0; i < 6; i++) out.put(e0 + 3 + i, es[i], poff + (uint32_t)i * WP);
    } else {
      // aggregatePointAdd (pointAdd.ts:199-259): C1..C6 = PX QX RX PY QY RY, at row slot (k % 3) * 2 + k / 3
      TomPt p[6];
      uint32_t x[PGL], y[PGL];
#pragma unroll
      for (int k = 0; k < 6; k++) { tom_parse(x, y, row + (size_t)((k % 3) * 2 + k / 3) * WP); tom_from_affine(p[k], x, y); }
      uint8_t der[DERS_PER_ITEM * BSTRIDE];
      point_add_derived(DerivedBytes{der}, p[0], p[1], p[2], p[3], p[4], p[5]);
      uint32_t chal[HASHES_PER_ITEM][3], a[PA_NCOM][8], in[6][8];
      for (int h = 0; h < HASHES_PER_ITEM; h++) pa_challenge(chal[h], h, der, tg_bytes, proof);
      fold_point_add(f, a, chal[0], proof, dr, out, e0 + 6, poff);
      point_add_expand(in, a);
#pragma unroll
      for (int k = 0; k < 6; k++) {
        const int slot = (k % 3) * 2 + k / 3;
        out.put_m(e0 + slot, in[k], (uint32_t)slot * WP);
      }
    }
    if (good && !f.tape_ok) ZK_SET_STATUS(status + b, ZKA_ERR_TAPE_RANGE);
    uint32_t v[8];
    zero_n<8>(v);
    st<8>(fx_jv + (size_t)b * 16, v); st<8>(fx_jr + (size_t)b * 16, v);
    F::from_mont(v, f.gW); st<8>(fx_jv + (size_t)b * 16 + 8, v);
    F::from_mont(v, f.hW); st<8>(fx_jr + (size_t)b * 16 + 8, v);
  }
};
struct VSubFinalTask {
  int32_t* status;
  const uint8_t* id_flags;   // [B][3], verdict at [b][1]
  uint8_t* ok;
  ZK_HD void operator()(int b) const { ok[b] = (status[b] == ZKA_OK && id_flags[(size_t)b * 3 + 1]) ? 1 : 0; }
};
struct VConcatTask {   // rows[b] = a[b] (la bytes) || c[b] (lc bytes)
  const uint8_t *a, *c;
  int la, lc;
  uint8_t* rows;
  size_t stride;
  ZK_HD void operator()(int t) const {
    const int per = la + lc;
    const int b = t / per, o = t % per;
    rows[(size_t)b * stride + o] = o < la ? a[(size_t)b * la + o] : c[(size_t)b * lc + (o - la)];
  }
};

// final verdict (zkpAttestList.ts:165-183): GK first, then exp
struct VFinalTask {
  VerifyCtx c;
  ZK_HD void operator()(int b) const {
    const uint8_t* fl = c.id_flags + (size_t)b * 3;
    // the aggregate check of the chunk stands for every per-proof identity test of its group (zk_verify_agg.cuh)
    const bool tom_pass = c.agg_ctl && c.agg_ctl[AGG_TOM_PASS], nist_pass = c.agg_ctl && c.agg_ctl[AGG_NIST_PASS];
    const bool f[3] = {tom_pass || fl[0], tom_pass || fl[1], nist_pass || fl[2]};
    const bool gk = c.gk_ok_len[b] && f[0];
    c.ok[b] = 0;
    // MALFORMED, R at infinity, a GK draw out of range: thrown before verifyMembership can return false
    if (c.status[b] != ZKA_OK) return;
    // verifyMembership returned false before verifyExp could throw: not an error
    if (!gk) return;
    const int key = c.vkey[b];
    if (key != VK_NONE) c.status[b] = key & 15;
    else c.ok[b] = (f[1] && f[2]) ? 1 : 0;
  }
};

}  // namespace zk
