// zk_trace.cuh — traceable proofs (include/zkattest.h, "Traceable proofs"; restated in tests/trace_rule.py).
//
// A traced row is the untraced proof followed by a trace block C1 C2 A0 A1 A2 s_x s_r s_k: a sigma proof that
// (C1, C2) = (k g, x g + k Y) encrypts the signer's key x "in the exponent" to the opener key Y = sk g, and that x is the
// value keyXcom = x g + r h commits to.  The stages below run after the batched prove / verify passes, never inside them;
// they see a row through its header (R comS1 keyXcom keyYcom, HEAD_LEN bytes) and its block, both staged per chunk.
// Fixed-base products are jobs of TomCommitTask (xyz form, so that pg_fixed_to_msm makes them group points); the products
// on Y, keyXcom, C1 and C2 are variable-base (pg_mul_var).  Written against the proof-group interface of zk_curves.cuh,
// so the tomEdwards256 and war256 builds compile from this one source.
#pragma once
#include "zk_seed.cuh"

namespace zk {

enum : int { TRACE_PTS = 5, TRACE_SCALARS = 3, TRACE_LEN = TRACE_PTS * WP + TRACE_SCALARS * WS, TRACE_DRAWS = 4 };
enum : uint32_t { SEED_DOM_TRACE = 4 };

// r = k P for a canonical k < 2^256: 65 signed 4-bit digits in [-7, 8] over the complete group law.  Every table entry
// is read for every digit (a select, not an index), so the memory accesses do not depend on a secret scalar.
ZK_HD void pg_mul_var(TomPt& r, const TomPt& P, const uint32_t* k) {
  constexpr int W = (int)(sizeof(TomPt) / sizeof(uint32_t));
  TomPt tab[8];
  tab[0] = P;
  tom_dbl(tab[1], P);
  for (int i = 2; i < 8; i++) tom_add(tab[i], tab[i - 1], P);
  int8_t d[65];
  uint32_t carry = 0;
  for (int i = 0; i < 64; i++) {
    const uint32_t v = ((k[i >> 3] >> (4 * (i & 7))) & 15u) + carry;
    carry = v > 8 ? 1u : 0u;
    d[i] = (int8_t)(carry ? (int)v - 16 : (int)v);
  }
  d[64] = (int8_t)carry;
  tom_set_identity(r);
  for (int i = 64; i >= 0; i--) {
    if (i < 64)
      for (int j = 0; j < 4; j++) tom_dbl(r, r);
    const int a = d[i] < 0 ? -d[i] : d[i];
    TomPt s, n;
    tom_set_identity(s);
    uint32_t* sw = reinterpret_cast<uint32_t*>(&s);
    for (int j = 1; j <= 8; j++) csel_n<W>(sw, a == j, reinterpret_cast<const uint32_t*>(&tab[j - 1]), sw);
    tom_neg(n, s);
    csel_n<W>(sw, d[i] < 0, reinterpret_cast<const uint32_t*>(&n), sw);
    tom_add(r, r, s);
  }
}

// a proof-group point from its encoding (validity is the caller's business)
ZK_HD void trace_point(TomPt& p, const uint8_t* b) {
  uint32_t x[PGL], y[PGL];
  tom_parse(x, y, b);
  tom_from_affine(p, x, y);
}
// a fixed-base job of TomCommitTask{xyz = 1} as a group point
ZK_HD void trace_fixed(TomPt& p, const uint32_t* proj) {
  tom_ld_xyz(p.x, p.y, p.z, proj);
  pg_fixed_to_msm(p);
}
ZK_HD void trace_put_scalar(uint8_t* o, const uint32_t* s) {
  if (WS == 33) o[0] = 0;
  limbs_to_be<8>(o + (WS - 32), s, 32);
}
// e = SHA-256("ZKAttest/trace/v1" || params digest || Y || msg_hash || header || C1 C2 A0 A1 A2), big-endian, mod q
ZK_HD void trace_challenge(uint32_t* e, const uint32_t* digest, const uint8_t* y, const uint8_t* msg, const uint8_t* hdr,
                           const uint8_t* pts) {
  Sha256 h;
  h.init();
  sha_tag(h, "ZKAttest/trace/v1");
  for (int i = 0; i < 8; i++) h.put4(digest[i]);
  h.update(y, WP);
  h.update(msg, 32);
  h.update(hdr, HEAD_LEN);
  h.update(pts, TRACE_PTS * WP);
  uint32_t d[8];
  h.final256(d);
  for (int i = 0; i < 8; i++) e[i] = d[7 - i];
  reduce_once<FpP256>(e);
}
// the 64-bit sort key of an encoding (its last eight bytes) for the opener's search
ZK_HD uint64_t trace_key(const uint8_t* b) {
  uint64_t k = 0;
  for (int i = WP - 8; i < WP; i++) k = (k << 8) | b[i];
  return k;
}

// ---- prover -------------------------------------------------------------------------------------------------------
// One thread per row: the witness x (keyToInt of pk) and r (draw 1), the draws k, a, beta, c, and the five fixed-base
// jobs (k, 0) (x, 0) (a, beta) (c, 0) (a, 0).  Tape draws: r at r_off and the four trace draws at t_off of each tape row;
// seeded rows: stream(seed, 1, 1) and stream(seed, 4, t), each rnd(q).  tstat = the row's status after its draws: the
// untraced status, else ZKA_ERR_TAPE_RANGE for a tape draw >= q.  A rejected row gets zero jobs.
struct TraceJobsTask {
  const int32_t* status;   // [B] untraced status
  const uint8_t* pk;       // [B][65]
  const uint8_t* tape;     // [B][tape_stride] or null
  size_t tape_stride, r_off, t_off;
  const uint8_t* seeds;    // [B][32] or null
  uint32_t *jv, *jr;       // [B][5][8]
  uint32_t* sec;           // [B][6][8] canonical x r k a beta c
  int32_t* tstat;          // [B]
  ZK_HD void operator()(int b) const {
    uint32_t s[6][8];
    bool range_ok = true;
    limbs_from_be<8>(s[0], pk + (size_t)b * 65 + 1, 32);
    reduce_once<FpP256>(s[0]);
    if (seeds) {
      uint32_t key[8], m[8], w[8];
      seed_key(key, seeds + (size_t)b * 32);
      seed_modulus(m, false);
      for (int t = 0; t <= TRACE_DRAWS; t++) {
        seed_draw32(w, key, t == 0 ? (uint32_t)SEED_DOM_PROVE : (uint32_t)SEED_DOM_TRACE, t == 0 ? 1u : (uint64_t)(t - 1), m);
        for (int i = 0; i < 8; i++) s[1 + t][7 - i] = bswap32(w[i]);
      }
    } else {
      const uint8_t* row = tape + (size_t)b * tape_stride;
      limbs_from_be<8>(s[1], row + r_off, 32);
      for (int t = 0; t < TRACE_DRAWS; t++) {
        limbs_from_be<8>(s[2 + t], row + t_off + 32 * t, 32);
        range_ok = lt_p<FpP256>(s[2 + t]) && range_ok;
      }
    }
    int32_t code = status[b];
    if (code == ZKA_OK && !range_ok) code = ZKA_ERR_TAPE_RANGE;
    tstat[b] = code;
    if (code != ZKA_OK)
      for (int i = 0; i < 6; i++) zero_n<8>(s[i]);
    for (int i = 0; i < 6; i++) st<8>(sec + ((size_t)b * 6 + i) * 8, s[i]);
    uint32_t z[8];
    zero_n<8>(z);
    const uint32_t* v[5] = {s[2], s[0], s[3], s[5], s[3]};
    const uint32_t* r[5] = {z, z, s[4], z, z};
    for (int j = 0; j < 5; j++) {
      st<8>(jv + ((size_t)b * 5 + j) * 8, v[j]);
      st<8>(jr + ((size_t)b * 5 + j) * 8, r[j]);
    }
  }
};
// One thread per (row, point): C1 = k g, C2 = x g + k Y, A0 = a g + beta h, A1 = c g, A2 = a g + c Y as E1 (X : Y : Z)
// for TomNormTask{e2 = 0}
struct TracePointsTask {
  const uint32_t* cproj;   // [B * 5][TOM_PROJ_WORDS] the jobs of TraceJobsTask
  const uint32_t* sec;     // [B][6][8]
  const uint8_t* y_bytes;  // [WP]
  uint32_t* pproj;         // [B * 5][TOM_PROJ_WORDS]
  ZK_HD void operator()(int t) const {
    const int b = t / TRACE_PTS, i = t % TRACE_PTS;
    TomPt f;
    trace_fixed(f, cproj + (size_t)t * TOM_PROJ_WORDS);
    if (i == 1 || i == 4) {
      TomPt Y, m;
      trace_point(Y, y_bytes);
      uint32_t s[8];
      ld<8>(s, sec + ((size_t)b * 6 + (i == 1 ? 2 : 5)) * 8);
      pg_mul_var(m, Y, s);
      tom_add(f, f, m);
    }
    tom_st_xyz(pproj + (size_t)t * TOM_PROJ_WORDS, f.x, f.y, f.z);
  }
};
// One thread per row: the war256 identity check (no encoding in a fixed slot), the challenge, s_x = a + e x,
// s_r = beta + e r, s_k = c + e k, and the block.  A rejected row's block is zero.
struct TraceFinishTask {
  uint32_t digest[8];      // the params digest as little-endian words in memory order
  const uint8_t* y_bytes;  // [WP]
  const uint8_t* msg_hash; // [B][32]
  const uint8_t* hdr;      // [B][HEAD_LEN]
  const uint8_t* pbytes;   // [B * 5][BSTRIDE]
  const uint32_t* sec;     // [B][6][8]
  int32_t* tstat;          // [B]
  uint8_t* blk;            // [B][TRACE_LEN]
  ZK_HD void operator()(int b) const {
    using F = Tomq;
    uint8_t* o = blk + (size_t)b * TRACE_LEN;
    const uint8_t* pb = pbytes + (size_t)b * TRACE_PTS * BSTRIDE;
    int32_t code = tstat[b];
    for (int i = 0; i < TRACE_PTS; i++)
      if (code == ZKA_OK && pb[(size_t)i * BSTRIDE] != 0x04) code = ZKA_ERR_IDENTITY_ENC;
    tstat[b] = code;
    if (code != ZKA_OK) {
      for (int i = 0; i < TRACE_LEN; i++) o[i] = 0;
      return;
    }
    for (int i = 0; i < TRACE_PTS; i++)
      for (int j = 0; j < WP; j++) o[i * WP + j] = pb[(size_t)i * BSTRIDE + j];
    uint32_t e[8], em[8];
    trace_challenge(e, digest, y_bytes, msg_hash + (size_t)b * 32, hdr + (size_t)b * HEAD_LEN, o);
    F::to_mont(em, e);
    const uint32_t* s = sec + (size_t)b * 48;
    for (int q = 0; q < TRACE_SCALARS; q++) {   // secrets x r k (0..2), nonces a beta c (3..5)
      uint32_t w[8], nn[8], t[8];
      ld<8>(w, s + 8 * q);
      ld<8>(nn, s + 8 * (3 + q));
      F::mul(t, em, w);
      F::add(t, nn, t);
      trace_put_scalar(o + TRACE_PTS * WP + q * WS, t);
    }
  }
};

// ---- check (verifier, the prover's self-check, the opener) ---------------------------------------------------------
// One thread per row: parse the block (the base parser's rules; a short row counts as unparsable), the challenge, and
// the fixed-base jobs (s_x, s_r) (s_k, 0) (s_x, 0) of the three relations
//   s_x g + s_r h = A0 + e keyXcom      s_k g = A1 + e C1      s_x g + s_k Y = A2 + e C2
struct TraceVJobsTask {
  uint32_t digest[8];
  const uint8_t* y_bytes;  // [WP]
  const uint8_t* msg_hash; // [B][32]
  const uint8_t* hdr;      // [B][HEAD_LEN]
  const uint8_t* blk;      // [B][TRACE_LEN]
  const uint8_t* shortrow; // [B] or null: 1 = proof_len < TRACE_LEN
  uint32_t *jv, *jr;       // [B][3][8]
  uint32_t* sc;            // [B][4][8] canonical e s_x s_r s_k
  uint8_t* bad;            // [B]
  ZK_HD void operator()(int b) const {
    const uint8_t* o = blk + (size_t)b * TRACE_LEN;
    bool ok = valid_points(o, TRACE_PTS);
    uint32_t s[4][8];
    for (int q = 0; q < TRACE_SCALARS; q++) ok = wscalar_parse(s[1 + q], o + TRACE_PTS * WP + q * WS) && ok;
    if (shortrow && shortrow[b]) ok = false;
    if (!ok)
      for (int q = 1; q < 4; q++) zero_n<8>(s[q]);
    trace_challenge(s[0], digest, y_bytes, msg_hash + (size_t)b * 32, hdr + (size_t)b * HEAD_LEN, o);
    bad[b] = ok ? 0 : 1;
    for (int q = 0; q < 4; q++) st<8>(sc + ((size_t)b * 4 + q) * 8, s[q]);
    uint32_t z[8];
    zero_n<8>(z);
    const uint32_t* v[3] = {s[1], s[3], s[1]};
    const uint32_t* r[3] = {s[2], z, z};
    for (int j = 0; j < 3; j++) {
      st<8>(jv + ((size_t)b * 3 + j) * 8, v[j]);
      st<8>(jr + ((size_t)b * 3 + j) * 8, r[j]);
    }
  }
};
// One thread per (row, relation): rel_ok = 1 when it holds
struct TraceVCheckTask {
  const uint32_t* cproj;   // [B * 3][TOM_PROJ_WORDS] the jobs of TraceVJobsTask
  const uint8_t* hdr;      // [B][HEAD_LEN]
  const uint8_t* blk;      // [B][TRACE_LEN]
  const uint8_t* y_bytes;  // [WP]
  const uint32_t* sc;      // [B][4][8]
  uint8_t* rel_ok;         // [B * 3]
  ZK_HD void operator()(int t) const {
    const int b = t / 3, i = t % 3;
    const uint8_t* o = blk + (size_t)b * TRACE_LEN;
    TomPt L, A, P, m;
    trace_fixed(L, cproj + (size_t)t * TOM_PROJ_WORDS);
    uint32_t s[8];
    if (i == 2) {
      TomPt Y;
      trace_point(Y, y_bytes);
      ld<8>(s, sc + ((size_t)b * 4 + 3) * 8);
      pg_mul_var(m, Y, s);
      tom_add(L, L, m);
    }
    trace_point(A, o + (size_t)(2 + i) * WP);
    trace_point(P, i == 0 ? hdr + (size_t)b * HEAD_LEN + 2 * NP : o + (size_t)(i - 1) * WP);
    ld<8>(s, sc + (size_t)b * 32);
    pg_mul_var(m, P, s);
    tom_add(A, A, m);
    tom_neg(A, A);
    tom_add(L, L, A);
    rel_ok[t] = pg_is_identity(L) ? 1 : 0;
  }
};
// The prover's self-check of its own blocks: a row the untraced pass accepted whose block fails becomes
// ZKA_ERR_SELF_CHECK.  chk[b]: 0 = not checked, 1 = passed, 2 = failed.
struct TraceSelfCheckTask {
  const uint8_t *bad, *rel_ok;
  int32_t* tstat;
  uint8_t* chk;
  ZK_HD void operator()(int b) const {
    if (tstat[b] != ZKA_OK) { chk[b] = 0; return; }
    const bool pass = !bad[b] && rel_ok[3 * b] && rel_ok[3 * b + 1] && rel_ok[3 * b + 2];
    chk[b] = pass ? 1 : 2;
    if (!pass) tstat[b] = ZKA_ERR_SELF_CHECK;
  }
};
// The verdict of a traced row from the untraced verdict (ok / status, in place): a block that does not parse is
// ZKA_ERR_MALFORMED, otherwise an accepted row also needs the three relations
struct TraceVerdictTask {
  const uint8_t *bad, *rel_ok;
  uint8_t* ok;
  int32_t* status;
  ZK_HD void operator()(int b) const {
    if (bad[b]) { ok[b] = 0; status[b] = ZKA_ERR_MALFORMED; return; }
    if (status[b] != ZKA_OK) { ok[b] = 0; return; }
    ok[b] = (ok[b] && rel_ok[3 * b] && rel_ok[3 * b + 1] && rel_ok[3 * b + 2]) ? 1 : 0;
  }
};

// Header and block of each row of a chunk of device rows; shortrow[b] = 1 when proof_len < TRACE_LEN
struct TraceGatherTask {
  const uint8_t* proofs;
  size_t stride;
  const uint32_t* len;     // [B]
  uint8_t *hdr, *blk, *shortrow;
  ZK_HD void operator()(int b) const {
    const uint8_t* row = proofs + (size_t)b * stride;
    const uint32_t l = len[b];
    const bool sh = l < (uint32_t)TRACE_LEN || (size_t)l > stride;
    shortrow[b] = sh ? 1 : 0;
    for (int i = 0; i < HEAD_LEN; i++) hdr[(size_t)b * HEAD_LEN + i] = (size_t)i < stride ? row[i] : 0;
    for (int i = 0; i < TRACE_LEN; i++) blk[(size_t)b * TRACE_LEN + i] = sh ? 0 : row[l - TRACE_LEN + i];
  }
};
// The blocks into device rows: row b gets blk[b] at byte off[b] (off < 0: the row is left as it is)
struct TraceApplyTask {
  uint8_t* proofs;
  size_t stride;
  const uint8_t* blk;
  const int64_t* off;      // [B]
  ZK_HD void operator()(int b) const {
    if (off[b] < 0) return;
    uint8_t* d = proofs + (size_t)b * stride + (size_t)off[b];
    for (int i = 0; i < TRACE_LEN; i++) d[i] = blk[(size_t)b * TRACE_LEN + i];
  }
};

// ---- opener ---------------------------------------------------------------------------------------------------------
// One thread per ring entry: the job (ring[j] mod q, 0) of (ring[j] mod q) g
struct TraceRingJobsTask {
  const uint8_t* ring;     // [N][32]
  uint32_t *jv, *jr;       // [N][8]
  ZK_HD void operator()(int j) const {
    uint32_t a[8];
    limbs_from_be<8>(a, ring + (size_t)j * 32, 32);
    reduce_once<FpP256>(a);
    st<8>(jv + (size_t)j * 8, a);
    zero_n<8>(a);
    st<8>(jr + (size_t)j * 8, a);
  }
};
// One thread per point: a TomCommitTask{xyz = 1} result as E1 (X : Y : Z), in place, for TomNormTask{e2 = 0}
struct TraceToE1Task {
  uint32_t* proj;          // [count][TOM_PROJ_WORDS]
  ZK_HD void operator()(int t) const {
    TomPt p;
    trace_fixed(p, proj + (size_t)t * TOM_PROJ_WORDS);
    tom_st_xyz(proj + (size_t)t * TOM_PROJ_WORDS, p.x, p.y, p.z);
  }
};
struct TraceKeyTask {      // one thread per ring entry: its sort key and index
  const uint8_t* bytes;    // [N][BSTRIDE]
  uint64_t* key;
  uint32_t* idx;
  ZK_HD void operator()(int j) const {
    key[j] = trace_key(bytes + (size_t)j * BSTRIDE);
    idx[j] = (uint32_t)j;
  }
};
// One thread per row: D = C2 - sk C1 as E1 (X : Y : Z)
struct TraceOpenDTask {
  uint32_t sk[8];
  const uint8_t* blk;      // [B][TRACE_LEN]
  uint32_t* dproj;         // [B][TOM_PROJ_WORDS]
  ZK_HD void operator()(int b) const {
    const uint8_t* o = blk + (size_t)b * TRACE_LEN;
    TomPt c1, c2, m;
    trace_point(c1, o);
    trace_point(c2, o + WP);
    pg_mul_var(m, c1, sk);
    tom_neg(m, m);
    tom_add(c2, c2, m);
    tom_st_xyz(dproj + (size_t)b * TOM_PROJ_WORDS, c2.x, c2.y, c2.z);
  }
};
// One thread per row: the smallest ring index whose point encodes as D.  The ring is sorted by key (a stable sort of
// the indices, so equal keys keep index order); the first entry with the key of D whose full encoding matches is the
// answer.  Precedence: ZKA_ERR_MALFORMED, ZKA_ERR_TRACE_INVALID, then the search (ZKA_ERR_NOT_IN_RING).
struct TraceFindTask {
  const uint8_t *bad, *rel_ok;
  const uint8_t* dbytes;   // [B][BSTRIDE]
  const uint8_t* rbytes;   // [N][BSTRIDE]
  const uint64_t* key;     // [N] sorted
  const uint32_t* idx;     // [N] in key order
  uint32_t N;
  uint32_t* index;         // [B]
  int32_t* status;         // [B]
  ZK_HD void operator()(int b) const {
    index[b] = 0xFFFFFFFFu;
    if (bad[b]) { status[b] = ZKA_ERR_MALFORMED; return; }
    if (!(rel_ok[3 * b] && rel_ok[3 * b + 1] && rel_ok[3 * b + 2])) { status[b] = ZKA_ERR_TRACE_INVALID; return; }
    const uint8_t* d = dbytes + (size_t)b * BSTRIDE;
    const uint64_t k = trace_key(d);
    uint32_t lo = 0, hi = N;
    while (lo < hi) {
      const uint32_t mid = lo + ((hi - lo) >> 1);
      if (key[mid] < k) lo = mid + 1; else hi = mid;
    }
    for (uint32_t p = lo; p < N && key[p] == k; p++) {
      const uint8_t* e = rbytes + (size_t)idx[p] * BSTRIDE;
      bool eq = true;
      for (int i = 0; i < WP; i++) eq = eq && e[i] == d[i];
      if (eq) { index[b] = idx[p]; status[b] = ZKA_OK; return; }
    }
    status[b] = ZKA_ERR_NOT_IN_RING;
  }
};

}  // namespace zk
