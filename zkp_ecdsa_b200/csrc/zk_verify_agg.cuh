// zk_verify_agg.cuh — chunk-wide aggregate check of the verifier ("all proofs of the chunk at once").
//
// verifySignatureList (/root/reference/src/zkpAttestList.ts:147-184) answers `isIdentity()` of three linear
// combinations per proof (GK, multiW, multiN; /root/reference/src/curves/multimult.ts:147-174 gives every relation of a
// proof its own random scalar drawn from the verify tape).  The tape is an input: rows of one call may share a tape row
// or a seed, and a prover may know it, so the tape scalars of DIFFERENT rows (or of GK and multiW of one row) need not be
// independent — two rejected rows whose residuals cancel would pass an unweighted sum.  Each combination of each row is
// therefore scaled by a weight of its own before the sums (AggWeightTask):
//
//     sum_b (wG_b GK_b + wW_b W_b) == O  and  sum_b wN_b N_b == O      <=>  (w.h.p.)  every single combination is O.
//
// The weights are 128-bit values from SHA-256 over the row's index in the call, the index of its ring, its message, its
// tape row and the proof bytes the verifier reads.  They change with every proof byte a residual depends on, so a
// prover cannot pick one row's residual after seeing that row's weight, and the index separates rows that share
// everything else; the argument needs no property of the tape beyond the reference's own.  Two limits: a weight
// depends on its own row only, so a prover who knows the tapes and controls k rows of a chunk can search for rows whose
// weighted residuals sum to O (a k-list birthday problem, about k 2^(256 / (1 + lg k)) hashes: 2^36 for k = 256) —
// but with a known tape it can forge each row against the reference's own per-row check directly, so this adds no
// weakness beyond the reference's; and the ring's keys, like the tape, are the verifier's input and are not hashed.
// The weights are odd (non-zero mod both prime orders) and the per-proof path never sees them.
//
// The per-proof evaluation (zk_verify.cuh: one thread per (proof, 6-bit window), 43 x (n_b + 64) point operations with
// n_b ~ 375) is therefore needed only when a sum is NOT the identity.  Each sum is ONE multi-scalar
// multiplication over all variable points of the chunk (~1.5 M tomEdwards256 points for 4096 proofs), evaluated with
// wide windows: signed c-bit digits (c = 12..16), counting sort of the entries by bucket, one thread per (window,
// bucket) summing its entries in registers, and a tree of weighted running sums over the buckets:
// ceil(258/c) x (n + 2^c) point operations for the whole chunk, 3-4x fewer than the per-proof windows.
//
//   pass:  every proof of the chunk is accepted (ok = 1) and the per-proof MSM kernels return at once;
//   fail (some proof is wrong, or some proof was already rejected by the parsers): the per-proof kernels run
//          exactly as before, so every verdict and status is the one the per-proof path gives.
// The verdict of a VALID batch is unchanged; for an invalid proof the per-proof path decides, under the same tape.
// tomEdwards256 has cofactor 4: a chunk in which some combination of some proof keeps a small-order component also goes
// to the per-proof path (AggTorsionTask), because the sums only vouch for the prime-order parts.
#pragma once
#include <string.h>

#include <cmath>

#include "zk_verify.cuh"

namespace zk {

#if defined(__CUDA_ARCH__)
ZK_HD uint32_t zk_atomic_add(uint32_t* p, uint32_t v) { return atomicAdd(p, v); }
#else
inline uint32_t zk_atomic_add(uint32_t* p, uint32_t v) { const uint32_t o = *p; *p = o + v; return o; }
#endif

enum : int {
  AGG_SEG = 256,      // buckets per segment of the prefix sum
  AGG_MAX_LEVELS = 6,
  AGG_FAN_BITS = 3,   // log2 of the largest fan-in of a reduction level (short latency chains: 7 x 3 additions)
  AGG_PIECE = 2048,   // bytes of tape per leaf of a row's digest tree
};

// ---- the rows' weights ---------------------------------------------------------------------------------------------
// A row's combinations depend on its message, ring and tape row and on the proof bytes the verifier reads: the header,
// the tag bits, every repetition's A, Tx, Ty (only through the exp challenge, whose full SHA-256 VChallengeTask keeps),
// the sampled repetitions and the GK block.  A row's digest is SHA-256 over a domain tag, its index in the call, its
// ring, its message, its tag bits, the challenge digest, its header and the digests of the pieces: AGG_PIECE-byte pieces
// of its tape row, each sampled repetition, the GK block (a two-level tree: the pieces hash in parallel).  Bytes the
// verifier never reads (the unsampled repetitions' responses) cannot move a residual and are left out.  Weight j = the
// first 128 bits of SHA-256(digest || j), made odd, in Montgomery form mod the group order of its combination: odd and
// below 2^128, so non-zero mod tom.order and mod p256.n.
ZK_HD int agg_tape_pieces(size_t tape_len) { return (int)((tape_len + AGG_PIECE - 1) / AGG_PIECE); }
struct AggPieceTask {   // one thread per (row, piece): tp tape pieces, K sampled repetitions, the GK block
  VerifyCtx c;
  size_t tape_len;
  int tp, np;           // np = tp + K + 1
  uint32_t* dig;        // [B][np][8]
  ZK_HD void operator()(int t) const {
    const int b = t / np, j = t % np;
    const uint32_t plen = c.proof_len[b] < c.proof_stride ? c.proof_len[b] : (uint32_t)c.proof_stride;
    const uint8_t* p;
    long lo, hi;
    if (j < tp) {
      p = c.tape_of(b);
      lo = (long)j * AGG_PIECE;
      hi = lo + AGG_PIECE < (long)tape_len ? lo + AGG_PIECE : (long)tape_len;
    } else {
      // a row the parsers rejected never reaches the aggregate: its offsets (parked at 0) only have to stay in bounds
      p = c.proof_of(b);
      if (j < tp + c.K) {
        const int i = (int)c.samp_idx[(size_t)b * c.K + (j - tp)];
        const uint32_t tag = (c.tagbits[(size_t)b * 3 + (i >> 5)] >> (i & 31)) & 1u;
        lo = c.rep_off[(size_t)b * c.S + i];
        hi = lo + (tag ? REP1_LEN : REP0_LEN);
      } else {
        lo = c.gk_off[b];
        hi = plen;
      }
      if (hi > (long)plen) hi = plen;
      if (lo > hi) lo = hi;
    }
    Sha256 h;
    h.init();
    h.update(p + lo, (int)(hi - lo));
    h.final256(dig + (size_t)t * 8);
  }
};
struct AggWeightTask {  // one thread per row
  VerifyCtx c;
  const uint32_t *chal_full, *dig;
  uint32_t row0;        // index in the call of the chunk's first row
  int np;
  uint32_t* wt;         // [B][AGG_WT][8]
  ZK_HD void operator()(int b) const {
    const uint32_t head[4] = {0x5741475au /* "ZGAW" */, row0 + (uint32_t)b, c.ring_of ? c.ring_of[b] : 0u, c.proof_len[b]};
    Sha256 h;
    h.init();
    h.update(reinterpret_cast<const uint8_t*>(head), (int)sizeof(head));
    h.update(c.msg_hash + (size_t)b * 32, 32);
    h.update(reinterpret_cast<const uint8_t*>(c.tagbits + (size_t)b * 3), 12);
    h.update(reinterpret_cast<const uint8_t*>(chal_full + (size_t)b * 8), 32);
    h.update(c.proof_of(b), c.proof_stride < HEAD_LEN ? (int)c.proof_stride : HEAD_LEN);
    h.update(reinterpret_cast<const uint8_t*>(dig + (size_t)b * np * 8), np * 32);
    uint32_t d[9];
    h.final256(d);
    for (int j = 0; j < AGG_WT; j++) {
      d[8] = (uint32_t)j;
      Sha256 g;
      g.init();
      g.update(reinterpret_cast<const uint8_t*>(d), 36);
      uint32_t o[8], w[8];
      g.final256(o);
      zero_n<8>(w);
      w[0] = o[3] | 1u;
      w[1] = o[2];
      w[2] = o[1];
      w[3] = o[0];
      if (j == AGG_W_N) P256n::to_mont(o, w);
      else Tomq::to_mont(o, w);
      st<8>(wt + ((size_t)b * AGG_WT + j) * 8, o);
    }
  }
};

// signed c-bit digits of a 256-bit scalar without a carry chain (see msm_digit6): with offs = sum_j 2^(c-1) 2^(c j)
// the unsigned windows of k + offs, minus 2^(c-1), are digits in [-2^(c-1), 2^(c-1)) whose weighted sum is k
//
// The TOP window holds only the bits of k above c (nwin - 1): its digit is non-negative and at most top_max =
// 2^(256 - c (nwin - 1)), so it would fill a handful of buckets with ~entries / top_max points each — one thread
// summing 10^5 points.  Its entries are therefore spread over
// 2^top_shift sub-buckets per digit, bucket index = (digit << top_shift) | (slot mod 2^top_shift); the reduction tree
// sums the sub-buckets without weights and weighs only the digit (AggLevelTask).
struct AggDigits {
  uint32_t offs[9];
  int c, nwin, nb;   // nb = 2^(c-1) buckets (|digit| = 1 .. nb)
  int top_shift;     // log2 sub-buckets per digit of the top window: (top_max + 1) << top_shift <= nb
};
// bucket (1 .. nb) of an entry: |digit| — for the top window the spread index + 1
ZK_HD uint32_t agg_bucket(const AggDigits& D, int w, int dabs, int slot) {
  if (w != D.nwin - 1) return (uint32_t)dabs;
  return (((uint32_t)dabs << D.top_shift) | ((uint32_t)slot & ((1u << D.top_shift) - 1u))) + 1u;
}
ZK_HD void agg_kp(uint32_t* kp, const uint32_t* k, const AggDigits& D) {
  uint64_t cy = 0;
#pragma unroll
  for (int i = 0; i < 9; i++) {
    cy += (uint64_t)(i < 8 ? k[i] : 0u) + D.offs[i];
    kp[i] = (uint32_t)cy;
    cy >>= 32;
  }
  kp[9] = 0;
}
ZK_HD int agg_digit(const uint32_t* kp, int w, int c) {   // kp[10]
  const int pos = w * c, wi = pos >> 5, sh = pos & 31;
  const uint64_t v = (uint64_t)kp[wi] | ((uint64_t)kp[wi + 1] << 32);
  return (int)((uint32_t)(v >> sh) & ((1u << c) - 1u)) - (1 << (c - 1));
}

// ---- host: the plan of one aggregate MSM ---------------------------------------------------------------------------
struct AggPlan {
  AggDigits D;
  int levels;
  int lm[AGG_MAX_LEVELS];   // log2 fan-in of every level of the bucket reduction (sum = c - 1)
};
// window bits from a cost model fitted to profiles/agg_window_sweep_r2i.md: ceil(258/c) windows x (entries / warp
// efficiency + 3 x 2^(c-1) bucket-tree additions); the warp efficiency accounts for the spread of the bucket sizes inside
// a warp (Poisson: about mean + sigma)
inline AggPlan agg_plan(double entries, int c_forced) {
  int best = 4;
  double best_cost = 1e300;
  for (int c = 4; c <= 16; c++) {
    const double nb = (double)(1u << (c - 1)), load = entries / nb;
    const double eff = load / (load + std::sqrt(load > 1.0 ? load : 1.0));
    const double cost = std::ceil(258.0 / c) * (entries / (eff > 0.05 ? eff : 0.05) + 3.0 * nb);
    if (cost < best_cost) { best_cost = cost; best = c; }
  }
  const int c = c_forced ? c_forced : best;
  AggPlan pl;
  memset(&pl, 0, sizeof(pl));
  pl.D.c = c;
  pl.D.nwin = (258 + c - 1) / c;
  pl.D.nb = 1 << (c - 1);
  for (int j = 0; j < pl.D.nwin; j++) {   // offs = sum_j 2^(c-1) 2^(c j)
    const int pos = c * j + c - 1;
    pl.D.offs[pos >> 5] |= 1u << (pos & 31);
  }
  // top window: digits 0 .. top_max, spread over 2^top_shift sub-buckets each
  const int tb = 256 - c * (pl.D.nwin - 1);
  const int top_max = 1 << (tb > 0 ? tb : 0);
  pl.D.top_shift = 0;
  while (((top_max + 1) << (pl.D.top_shift + 1)) <= pl.D.nb) pl.D.top_shift++;
  const int bits = c - 1;
  pl.levels = (bits + AGG_FAN_BITS - 1) / AGG_FAN_BITS;
  for (int i = 0; i < pl.levels; i++) pl.lm[i] = bits / pl.levels + (i < bits % pl.levels ? 1 : 0);
  return pl;
}

// ---- entry sources: slot -> (used?, scalar, point) ---------------------------------------------------------------
struct AggTomSrc {
  const uint32_t *ent_scalar, *ent_pre, *ent_cnt, *gk_scalar, *gk_pre;
  int B, ET, K, ngk;   // slots [0, B*ET): multiW entries (K samples x 34 + keyXcom, keyYcom); then B*ngk GK entries
  const uint32_t* wt;  // [B][AGG_WT][8] the rows' weights (AggWeightTask)
  using Pt = TomPt;
  enum { PTW = PG_EXT_WORDS };
  ZK_HD int slots() const { return B * (ET + ngk); }
  ZK_HD bool used(int s) const {
    if (s >= B * ET) return true;
    const int b = s / ET, e = s % ET;
    if (e >= K * V_ENT_PER_SAMPLE) return true;
    return (uint32_t)(e % V_ENT_PER_SAMPLE) < ent_cnt[(size_t)b * K + e / V_ENT_PER_SAMPLE];
  }
  ZK_HD const uint32_t* scalar(int s) const {
    return s < B * ET ? ent_scalar + (size_t)s * 8 : gk_scalar + (size_t)(s - B * ET) * 8;
  }
  // the scalar the aggregate MSM uses: times the weight of the slot's row and combination (multiW or GK)
  ZK_HD void load(uint32_t* k, int s) const {
    ld<8>(k, scalar(s));
    const bool w = s < B * ET;
    const int b = w ? s / ET : (s - B * ET) / ngk;
    uint32_t m[8];
    ld<8>(m, wt + ((size_t)b * AGG_WT + (w ? AGG_W_W : AGG_W_GK)) * 8);
    Tomq::mul(k, k, m);
  }
  ZK_HD void accumulate(Pt& acc, int s, bool neg) const {
    TomPre pt;
    tom_ld_pre(pt, s < B * ET ? ent_pre + (size_t)s * TOM_PRE_WORDS : gk_pre + (size_t)(s - B * ET) * TOM_PRE_WORDS);
    if (neg) pg_pre_neg(pt);
    tom_madd<true, TompMsm>(acc, acc, pt);
  }
  ZK_HD static void identity(Pt& p) { tom_set_identity(p); }
  ZK_HD static void add(Pt& r, const Pt& p, const Pt& q) { tom_add(r, p, q); }
  ZK_HD static void dbl(Pt& r, const Pt& p) { tom_dbl(r, p); }
  ZK_HD static void dbl_n(Pt& p, int c) { pg_dbl_n(p, c); }
  ZK_HD static void ld_pt(Pt& p, const uint32_t* m) { bk_load(p, reinterpret_cast<const U4*>(m)); }
  ZK_HD static void st_pt(uint32_t* m, const Pt& p) { bk_store(reinterpret_cast<U4*>(m), p); }
};
struct AggNistSrc {
  const uint32_t *scalar_, *aff;
  const uint8_t* skip;
  int B, EN;
  const uint32_t* wt;
  using Pt = P256Pt;
  enum { PTW = 24 };
  ZK_HD int slots() const { return B * EN; }
  ZK_HD bool used(int s) const { return skip[s] == 0; }
  ZK_HD const uint32_t* scalar(int s) const { return scalar_ + (size_t)s * 8; }
  ZK_HD void load(uint32_t* k, int s) const {
    ld<8>(k, scalar(s));
    uint32_t m[8];
    ld<8>(m, wt + ((size_t)(s / EN) * AGG_WT + AGG_W_N) * 8);
    P256n::mul(k, k, m);
  }
  ZK_HD void accumulate(Pt& acc, int s, bool neg) const {
    P256Aff q;
    p256_ld_aff(q, aff + (size_t)s * P256_AFF_WORDS);
    if (neg) P256p::neg(q.y, q.y);
    p256_madd(acc, acc, q);
  }
  ZK_HD static void identity(Pt& p) { p256_set_identity(p); }
  ZK_HD static void add(Pt& r, const Pt& p, const Pt& q) { p256_add(r, p, q); }
  ZK_HD static void dbl(Pt& r, const Pt& p) { p256_dbl(r, p); }
  ZK_HD static void dbl_n(Pt& p, int c) { p256_dbl_n(p, c); }
  ZK_HD static void ld_pt(Pt& p, const uint32_t* m) { p256_ld_proj(p, m); }
  ZK_HD static void st_pt(uint32_t* m, const Pt& p) { p256_st_proj(m, p); }
};

// A0 — is every proof of the chunk eligible?  (a proof the parsers already rejected keeps its per-proof verdict)
struct AggGateTask {
  VerifyCtx c;
  uint32_t* ctl;
  ZK_HD void operator()(int b) const {
    if (c.status[b] != ZKA_OK || c.vkey[b] != VK_NONE || (c.mode == 0 && !c.gk_ok_len[b])) ctl[AGG_SKIP] = 1;
  }
};

#if !defined(ZKA_PG_WAR256)
// A0b — tomEdwards256 has cofactor 4, and deserializePoint (edwards.ts:70-86) only checks the curve equation.  Points
// with a small-order component make the reference's own verdict depend on its randomizers (a component of order 2
// survives a relation iff its scalar is odd).  The weighted sums only vouch for the prime-order parts of the
// combinations, so the aggregate verdict is used only when no combination of any proof keeps a small-order component
// under the reference's OWN scalars (the unweighted ones: a weighted scalar is reduced mod q, which changes it mod 4).
// With tau the projection onto E[4],  tau(C) = sum_e (s_e mod 4) tau(P_e) = tau(W)  for  W = sum_e (s_e mod 4) P_e
// (fixed-base parts are multiples of g, h: prime order), and  q W = (q mod 4) tau(W) = -tau(W)  (q = p256.p = 3 mod 4).
// GK and multiW are checked apart: the reference rejects a row whose GK keeps a component that its multiW cancels.
// Then for every row  C = pi(C)  (pi: the prime-order part), and a weighted sum that is O has every pi(C) = O (w.h.p.).
// ~n_b mixed additions and 256 doublings per combination; q = 2^256 - 2^224 + 2^192 + 2^96 - 1 costs four more
// additions.  Two steps: partial sums per (proof, part) — parts 0..K-1 the sampled repetitions, part K keyXcom and
// keyYcom (multiW), part K + 1 the GK points — then one thread per (proof, combination) for the additions and the
// doubling chain.
struct AggTorsionPartTask {   // one thread per (proof, part, bit of s mod 4): ONE accumulator per thread (two spilled)
  AggTomSrc src;
  const uint32_t* ctl;
  uint32_t* part;    // [B][K + 2][2][PG_EXT_WORDS]: sums of the points with bit 0 / bit 1 of (s mod 4) set
  ZK_HD void add_range(TomPt& a, uint32_t mask, int s0, int cnt) const {
    for (int e = 0; e < cnt; e++) {
      const int s = s0 + e;
      if (!src.used(s)) continue;
      if (src.scalar(s)[0] & mask) src.accumulate(a, s, false);
    }
  }
  ZK_HD void operator()(int t) const {
    if (ctl[AGG_SKIP]) return;
    const int bit = t & 1, bj = t >> 1;
    const int b = bj / (src.K + 2), j = bj % (src.K + 2);
    const uint32_t mask = 1u << bit;
    TomPt a;
    tom_set_identity(a);
    if (j < src.K) add_range(a, mask, b * src.ET + j * V_ENT_PER_SAMPLE, V_ENT_PER_SAMPLE);
    else if (j == src.K) add_range(a, mask, b * src.ET + src.K * V_ENT_PER_SAMPLE, src.ET - src.K * V_ENT_PER_SAMPLE);
    else add_range(a, mask, src.B * src.ET + b * src.ngk, src.ngk);
    bk_store(reinterpret_cast<U4*>(part + (size_t)t * PG_EXT_WORDS), a);
  }
};
struct AggTorsionTask {   // one thread per (proof, combination): t = 2 b + (0: GK, 1: multiW)
  const uint32_t* part;
  uint32_t* ctl;
  int K;
  ZK_HD void operator()(int t) const {
    if (ctl[AGG_SKIP]) return;
    const int b = t >> 1;
    const int j0 = (t & 1) ? 0 : K + 1, j1 = (t & 1) ? K : K + 1;
    TomPt a1, a2, p;
    tom_set_identity(a1);
    tom_set_identity(a2);
    for (int j = j0; j <= j1; j++) {
      const uint32_t* o = part + ((size_t)b * (K + 2) + j) * 2 * PG_EXT_WORDS;
      bk_load(p, reinterpret_cast<const U4*>(o));
      tom_add(a1, a1, p);
      bk_load(p, reinterpret_cast<const U4*>(o + PG_EXT_WORDS));
      tom_add(a2, a2, p);
    }
    TomPt w, r;
    tom_dbl(a2, a2);
    tom_add(w, a1, a2);           // W
    TomPt tt = w;
    for (int i = 0; i < 96; i++) tom_dbl(tt, tt);
    tom_neg(r, w);
    tom_add(r, r, tt);            // 2^96 W - W
    for (int i = 96; i < 192; i++) tom_dbl(tt, tt);
    tom_add(r, r, tt);            // + 2^192 W
    for (int i = 192; i < 224; i++) tom_dbl(tt, tt);
    TomPt n;
    tom_neg(n, tt);
    tom_add(r, r, n);             // - 2^224 W
    for (int i = 224; i < 256; i++) tom_dbl(tt, tt);
    tom_add(r, r, tt);            // + 2^256 W
    if (!pg_is_identity(r)) ctl[AGG_SKIP] = 1;
  }
};
#endif

// A1 — histogram of |digit| per window.  One thread per slot.
template <class Src>
struct AggHistTask {
  Src src;
  AggDigits D;
  const uint32_t* ctl;
  uint32_t* hist;   // [nwin][nb + 1]
  ZK_HD void operator()(int s) const {
    if (ctl[AGG_SKIP] || !src.used(s)) return;
    uint32_t k[8], kp[10];
    src.load(k, s);
    agg_kp(kp, k, D);
    for (int w = 0; w < D.nwin; w++) {
      const int d = agg_digit(kp, w, D.c);
      if (d) zk_atomic_add(hist + (size_t)w * (D.nb + 1) + agg_bucket(D, w, d < 0 ? -d : d, s), 1u);
    }
  }
};
// A2 — exclusive prefix sums of the histogram rows, in three steps (segment totals, scan of the totals, offsets)
struct AggSegSumTask {
  const uint32_t *ctl, *hist;
  uint32_t* segtot;   // [nwin][nseg]
  int nb, nseg;
  ZK_HD void operator()(int t) const {
    if (ctl[AGG_SKIP]) return;
    const int w = t / nseg, sg = t % nseg;
    const uint32_t* h = hist + (size_t)w * (nb + 1);
    uint32_t sum = 0;
    for (int d = sg * AGG_SEG; d < (sg + 1) * AGG_SEG && d <= nb; d++) sum += h[d];
    segtot[t] = sum;
  }
};
struct AggSegScanTask {
  const uint32_t* ctl;
  uint32_t* segtot;
  int nseg;
  ZK_HD void operator()(int w) const {
    if (ctl[AGG_SKIP]) return;
    uint32_t run = 0;
    for (int i = 0; i < nseg; i++) {
      const uint32_t v = segtot[(size_t)w * nseg + i];
      segtot[(size_t)w * nseg + i] = run;
      run += v;
    }
  }
};
struct AggOffsetsTask {
  const uint32_t *ctl, *segtot;
  uint32_t* hist;     // in: counts; out: running cursor of each bucket (= its start)
  uint32_t* bstart;   // [nwin][nb + 2]: start of bucket d, bstart[nb + 1] = entries of the window
  int nb, nseg;
  ZK_HD void operator()(int t) const {
    if (ctl[AGG_SKIP]) return;
    const int w = t / nseg, sg = t % nseg;
    uint32_t* h = hist + (size_t)w * (nb + 1);
    uint32_t* bs = bstart + (size_t)w * (nb + 2);
    uint32_t run = segtot[t];
    for (int d = sg * AGG_SEG; d < (sg + 1) * AGG_SEG && d <= nb; d++) {
      const uint32_t v = h[d];
      h[d] = run;
      bs[d] = run;
      run += v;
      if (d == nb) bs[nb + 1] = run;
    }
  }
};
// A3 — scatter the slots into bucket order (sign in bit 31).  The order inside a bucket depends on the atomics; the
// bucket SUM does not (only the projective representation of it).
template <class Src>
struct AggScatterTask {
  Src src;
  AggDigits D;
  const uint32_t* ctl;
  uint32_t* cursor;   // [nwin][nb + 1]
  uint32_t* sorted;   // [nwin][cap]
  size_t cap;
  ZK_HD void operator()(int s) const {
    if (ctl[AGG_SKIP] || !src.used(s)) return;
    uint32_t k[8], kp[10];
    src.load(k, s);
    agg_kp(kp, k, D);
    for (int w = 0; w < D.nwin; w++) {
      const int d = agg_digit(kp, w, D.c);
      if (d) {
        const uint32_t pos = zk_atomic_add(cursor + (size_t)w * (D.nb + 1) + agg_bucket(D, w, d < 0 ? -d : d, s), 1u);
        sorted[(size_t)w * cap + pos] = (uint32_t)s | (d < 0 ? 0x80000000u : 0u);
      }
    }
  }
};
// A4 — bucket sums: one thread per (window, bucket), entries summed in registers.
template <class Src>
struct AggBucketTask {
  Src src;
  const uint32_t *ctl, *bstart, *sorted;
  uint32_t* bsum;   // [nwin][nb][PTW]
  size_t cap;
  int nb;
  ZK_HD void operator()(int t) const {
    if (ctl[AGG_SKIP]) return;
    const int w = t / nb, d = 1 + t % nb;
    const uint32_t* bs = bstart + (size_t)w * (nb + 2);
    const uint32_t lo = bs[d], hi = bs[d + 1];
    typename Src::Pt acc;
    Src::identity(acc);
    const uint32_t* so = sorted + (size_t)w * cap;
    for (uint32_t q = lo; q < hi; q++) {
      const uint32_t e = so[q];
      src.accumulate(acc, (int)(e & 0x7fffffffu), (e >> 31) != 0);
    }
    Src::st_pt(bsum + (size_t)t * Src::PTW, acc);
  }
};
#if !defined(ZKA_HOSTSIM) && defined(ZKA_MSM_MINBLOCKS)
template <> struct TaskMinBlocks<AggBucketTask<AggTomSrc>> { static constexpr int value = ZKA_MSM_MINBLOCKS; };
#endif
// A5 — one level of the weighted running sums.  A node covering bucket indices [lo, lo + len) holds
//   A = sum S_i   and   B = sum (i - lo) S_i ;
// m = 2^lm children of length l = 2^ll combine as  A' = sum_k A_k,  B' = sum_k B_k + l * sum_k k A_k, and
// sum_k k A_k is the classic running sum (run += A_k; tot += run, k = m-1 .. 1).  Leaves (ll = 0) have no B.
// Top window (spread buckets, weight of index i = i >> ts): child k weighs (k >> s) 2^max(ll - ts, 0) with
// s = clamp(ts - ll, 0, lm) — below the spread the sums are plain, above it the usual tree.
template <class Src>
struct AggLevelTask {
  const uint32_t *ctl, *inA, *inB;   // [nwin][nin][PTW]; inB null at the first level
  uint32_t *outA, *outB;             // [nwin][nin >> lm][PTW]
  int nin, lm, ll;
  int nwin, top_shift;
  ZK_HD void operator()(int t) const {
    if (ctl[AGG_SKIP]) return;
    using Pt = typename Src::Pt;
    const int nout = nin >> lm, m = 1 << lm;
    const int w = t / nout, node = t % nout;
    const int ts = w == nwin - 1 ? top_shift : 0;
    int s = ts - ll;
    s = s < 0 ? 0 : (s > lm ? lm : s);
    const int dbl = ll > ts ? ll - ts : 0;
    const bool useB = inB && ll > ts;      // the children carry weights of their own only above the spread
    const size_t base = ((size_t)w * nin + (size_t)node * m) * Src::PTW;
    Pt run, tot, sb, a;
    Src::identity(run);
    Src::identity(tot);
    Src::identity(sb);
    for (int k = m - 1; k >= 0; k--) {
      Src::ld_pt(a, inA + base + (size_t)k * Src::PTW);
      Src::add(run, run, a);
      if (k > 0 && (k & ((1 << s) - 1)) == 0) Src::add(tot, tot, run);   // sum_k (k >> s) A_k
      if (useB) {
        Src::ld_pt(a, inB + base + (size_t)k * Src::PTW);
        Src::add(sb, sb, a);
      }
    }
    if (dbl) Src::dbl_n(tot, dbl);
    Src::add(sb, sb, tot);
    Src::st_pt(outA + (size_t)t * Src::PTW, run);
    Src::st_pt(outB + (size_t)t * Src::PTW, sb);
  }
};
// window w total = sum_{d=1..nb} d S_d = B_root + A_root (bucket d sits at index d - 1); the spread top window weighs
// index i with i >> top_shift = its digit: B_root alone.  Result = sum_w 2^(c w) total_w.
template <class Src>
ZK_HD void agg_horner(typename Src::Pt& acc, const uint32_t* rootA, const uint32_t* rootB, int nwin, int c) {
  typename Src::Pt t, u;
  Src::identity(acc);
  for (int w = nwin - 1; w >= 0; w--) {
    Src::dbl_n(acc, c);
    Src::ld_pt(u, rootB + (size_t)w * Src::PTW);
    if (w != nwin - 1) {
      Src::ld_pt(t, rootA + (size_t)w * Src::PTW);
      Src::add(u, u, t);
    }
    Src::add(acc, acc, u);
  }
}

// ---- fixed-base parts -------------------------------------------------------------------------------------------
// tomEdwards256: sum_b (wG_b (v_b0 g + r_b0 h) + wW_b (v_b1 g + r_b1 h)) = (sum w v) g + (sum w r) h — the weighted
// SCALARS are summed (mod the group order) and ONE fixed-base commitment is evaluated for the whole chunk.
struct AggFixPartTask {   // one thread per group of 32 proofs
  const uint32_t *ctl, *fx_jv, *fx_jr;   // [B*2][8] canonical mod q (job 0: GK, job 1: multiW)
  const uint32_t* wt;                    // [B][AGG_WT][8]
  uint32_t* part;                        // [groups][2][8]
  int B;
  ZK_HD void operator()(int g) const {
    if (ctl[AGG_SKIP]) return;
    using F = Tomq;
    uint32_t sv[8], sr[8], t[8];
    zero_n<8>(sv);
    zero_n<8>(sr);
    uint32_t m[8];
    for (int i = g * 64; i < (g + 1) * 64 && i < B * 2; i++) {
      ld<8>(m, wt + ((size_t)(i >> 1) * AGG_WT + (i & 1)) * 8);   // job i & 1 = weight AGG_W_GK / AGG_W_W
      ld<8>(t, fx_jv + (size_t)i * 8); F::mul(t, t, m); F::add(sv, sv, t);
      ld<8>(t, fx_jr + (size_t)i * 8); F::mul(t, t, m); F::add(sr, sr, t);
    }
    st<8>(part + (size_t)g * 16, sv);
    st<8>(part + (size_t)g * 16 + 8, sr);
  }
};
struct AggFixSumTask {
  const uint32_t *ctl, *part;
  uint32_t *jv, *jr;   // [1][8]: the job of TomCommitTask
  int groups;
  ZK_HD void operator()(int) const {
    using F = Tomq;
    uint32_t sv[8], sr[8], t[8];
    zero_n<8>(sv);
    zero_n<8>(sr);
    for (int g = 0; g < (ctl[AGG_SKIP] ? 0 : groups); g++) {   // skipped chunk: the commitment job gets zeros
      ld<8>(t, part + (size_t)g * 16); F::add(sv, sv, t);
      ld<8>(t, part + (size_t)g * 16 + 8); F::add(sr, sr, t);
    }
    st<8>(jv, sv);
    st<8>(jr, sr);
  }
};
// P-256: sum_b wN_b (sR_b R_b + shN_b h) — R differs per proof, so the POINTS are summed: each row's weighted fixed part
// from its weighted scalars (the per-proof path keeps the unweighted nfix), then a tree of 32-way partial sums
struct AggNistFixWeightTask {   // one thread per proof
  const uint32_t *ctl, *k, *wt, *rtab, *h_tab8;   // k: [B][2][8] sR, shN (VReduceTask)
  int h_w;
  uint32_t* out;                                  // [B][24]
  ZK_HD void operator()(int b) const {
    if (ctl[AGG_SKIP]) return;
    uint32_t m[8], kR[8], kH[8];
    ld<8>(m, wt + ((size_t)b * AGG_WT + AGG_W_N) * 8);
    ld<8>(kR, k + (size_t)b * 16);
    ld<8>(kH, k + (size_t)b * 16 + 8);
    P256n::mul(kR, kR, m);
    P256n::mul(kH, kH, m);
    P256Pt acc;
    p256_set_identity(acc);
    p256_accum_rtab(acc, rtab + (size_t)b * RT_ENTRIES * P256_AFF_WORDS, kR);
    p256_accum_fixed(acc, h_tab8, kH, h_w);
    p256_st_proj(out + (size_t)b * P256_PROJ_WORDS, acc);
  }
};
struct AggNistFixPartTask {
  const uint32_t *ctl, *in;     // [count][24]
  uint32_t* part;               // [ceil(count / 32)][24]
  int count;
  ZK_HD void operator()(int g) const {
    if (ctl[AGG_SKIP]) return;
    P256Pt acc, p;
    p256_set_identity(acc);
    for (int i = g * 32; i < (g + 1) * 32 && i < count; i++) {
      p256_ld_proj(p, in + (size_t)i * P256_PROJ_WORDS);
      p256_add(acc, acc, p);
    }
    p256_st_proj(part + (size_t)g * P256_PROJ_WORDS, acc);
  }
};

// A6 — Horner over the windows, the fixed parts, the verdicts.  Thread 0: tomEdwards256, thread 32: P-256.
struct AggFinalTask {
  uint32_t* ctl;
  const uint32_t *tomA, *tomB, *fx_proj;   // roots [nwin][36] and the chunk's fixed-base commitment (E2 model, 28 words)
  int t_nwin, t_c;
  const uint32_t *nisA, *nisB, *nfix_part; // roots [nwin][24] and the partial sums of the fixed parts
  int n_nwin, n_c, n_groups;
  ZK_HD void operator()(int t) const {
    if (ctl[AGG_SKIP]) return;
    if (t == 0) {
      TomPt acc, f;
      agg_horner<AggTomSrc>(acc, tomA, tomB, t_nwin, t_c);
      tom_ld_xyz(f.x, f.y, f.z, fx_proj);
      pg_fixed_to_msm(f);
      tom_add(acc, acc, f);
      ctl[AGG_TOM_PASS] = pg_is_identity(acc) ? 1u : 0u;
    } else if (t == 32) {
      P256Pt acc, p;
      agg_horner<AggNistSrc>(acc, nisA, nisB, n_nwin, n_c);
      for (int g = 0; g < n_groups; g++) {
        p256_ld_proj(p, nfix_part + (size_t)g * P256_PROJ_WORDS);
        p256_add(acc, acc, p);
      }
      ctl[AGG_NIST_PASS] = p256_is_identity(acc) ? 1u : 0u;
    }
  }
};

}  // namespace zk
