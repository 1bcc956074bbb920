// zk_ops_war.cuh — proof-group tasks of the war256 build (included by zk_ops.cuh when ZKA_PG_WAR256 is defined).
//
// Same task names and fields as the tomEdwards256 versions in zk_ops.cuh, so the host pipelines in zkattest.cu launch
// them unchanged; the bodies work on war256 = short Weierstrass, a = -3 (/root/reference/src/curves/instances.ts:34-41,
// group law /root/reference/src/curves/weier.ts:133-230 — the second inclusion of zk_weier.inc / zk_weier_ops.inc):
//   * fixed-base tables are positional signed-digit tables of AFFINE points [fb_windows(w)][fb_entries(w)][16]
//     (entry 0 of a window is never read: a zero digit skips the addition, the identity has no affine form),
//   * a commitment v*g + r*h walks both tables with the complete mixed addition (RCB15 Alg. 5, 11M + 2 m_b),
//   * normalisation is one batched inversion per chunk and the SEC1 encoding 04 || x || y (weier.ts:244-255).
#pragma once

#define WEI_PT WarPt
#define WEI_AFF WarAff
#define WEI_JAC WarJac
#define WEI_F Warp
#define WEI_FN(n) war_##n
#define WEI_T(n) War##n
#include "zk_weier_ops.inc"
#undef WEI_PT
#undef WEI_AFF
#undef WEI_JAC
#undef WEI_F
#undef WEI_FN
#undef WEI_T

// Batched normalisation of war256 points -> affine Montgomery (x, y) (+ optional 65-byte encoding).  `e2` is the
// tomEdwards256 build's curve-model flag and is ignored here; the identity encodes as 65 zero bytes.
struct TomNormTask {
  const uint32_t* proj;  // [count][24]
  uint32_t* aff;         // [count][16] or null
  uint8_t* bytes;        // [count][BSTRIDE] or null
  int count;
  int chunk;             // points per thread (<= NORM_CHUNK_MAX)
  int e2;
  int aff_mod, aff_lim;  // the affine pair is produced only for points with (index % aff_mod) < aff_lim
  int stride;            // words per input slot (TOM_PROJ_WORDS = TOM_E2_WORDS)
  ZK_HD void operator()(int t) const {
    using F = Warp;
    const int lo = t * chunk;
    int n = count - lo;
    if (n > chunk) n = chunk;
    if (n <= 0) return;
    uint32_t pre[NORM_CHUNK_MAX][8];
    uint32_t acc[8], z[8], one[8];
    F::set_one(one);
    copy_n<8>(acc, one);
    for (int k = 0; k < n; k++) {
      ld<8>(z, proj + (size_t)(lo + k) * stride + 16);
      if (is_zero_n<8>(z)) copy_n<8>(z, one);
      F::mul(acc, acc, z);
      copy_n<8>(pre[k], acc);
    }
    uint32_t inv[8];
    F::inv(inv, acc);
    for (int k = n - 1; k >= 0; k--) {
      const uint32_t* src = proj + (size_t)(lo + k) * stride;
      ld<8>(z, src + 16);
      const bool isinf = is_zero_n<8>(z);
      if (isinf) copy_n<8>(z, one);
      uint32_t zi[8];
      if (k > 0) F::mul(zi, inv, pre[k - 1]); else copy_n<8>(zi, inv);
      F::mul(inv, inv, z);
      uint32_t X[8], Y[8], x[8], y[8];
      ld<8>(X, src);
      ld<8>(Y, src + 8);
      F::mul(x, X, zi);
      F::mul(y, Y, zi);
      if (aff && ((lo + k) % aff_mod) < aff_lim) {
        uint32_t* a = aff + (size_t)(lo + k) * TOM_AFF_WORDS;
        st<8>(a, x);
        st<8>(a + 8, y);
      }
      if (bytes) {
        uint32_t cx[8], cy[8];
        F::from_mont(cx, x);
        F::from_mont(cy, y);
        if (isinf) { zero_n<8>(cx); zero_n<8>(cy); }
        store_point_words<8, 32>(bytes + (size_t)(lo + k) * BSTRIDE, isinf ? 0x00u : 0x04u, cx, cy);
      }
    }
  }
};

// Pedersen commitment in the proof group:  C = v*g + r*h   (pedersen.ts:53-58, gk.ts:88-92).  Both walks run on one
// Jacobian accumulator that starts at the identity: jac_madd takes the first non-zero digit's entry as (x : y : 1)
// without products, as the tomEdwards256 walks start at their first entry.
struct TomCommitTask {
  const uint32_t* jv;    // [count][8] canonical value scalars (mod war256.order = p256.p)
  const uint32_t* jr;    // [count][8] canonical blinders
  const uint32_t* gtab;  // [nwin][E][16]
  const uint32_t* htab;
  uint32_t* proj;        // [count][24]
  FbShape sh;             // always uniform in this build: sh.w bits in every window
  int xyz = 0;           // the tomEdwards256 build's output-form flag; the output here is always (X, Y, Z)
  ZK_HD void operator()(int t) const {
    uint32_t v[8], r[8];
    ld<8>(v, jv + (size_t)t * 8);
    ld<8>(r, jr + (size_t)t * 8);
    WarJac aj;
    war_set_identity_jac(aj);
    war_accum_fixed_jac(aj, gtab, v, sh.w);
    war_accum_fixed_jac(aj, htab, r, sh.w);
    WarPt acc;
    war_jac_to_hom(acc, aj);
    war_st_proj(proj + (size_t)t * TOM_PROJ_WORDS, acc);
  }
};
// the jobs of a batch share g-parts as GpartLayout says (see zk_ops.cuh)
ZK_HD void war_gpart(WarPt& acc, const uint32_t* gtab, const uint32_t* v, int w) {   // v*g
  WarJac aj;
  war_set_identity_jac(aj);
  war_accum_fixed_jac(aj, gtab, v, w);
  war_jac_to_hom(acc, aj);
}
struct TomCommitGTask {   // one thread per g-part of GpartLayout: K = v*g
  const uint32_t* jv;     // [rows * lay.jobs()][8]
  const uint32_t* gtab;
  uint32_t* ext;          // [rows * lay.gparts()][24]
  FbShape sh;             // always uniform in this build: sh.w bits in every window
  GpartLayout lay;
  ZK_HD void operator()(int t) const {
    const int row = t / lay.gparts(), jb = lay.job_of_gpart(row, t % lay.gparts());
    if (jb < 0) return;
    uint32_t v[8];
    ld<8>(v, jv + ((size_t)row * lay.jobs() + jb) * 8);
    WarPt acc;
    war_gpart(acc, gtab, v, sh.w);
    war_st_proj(ext + (size_t)t * TOM_EXT_WORDS, acc);
  }
};
struct TomCommitHTask {   // one thread per job: C = K + r*h
  const uint32_t* jv;     // [rows * lay.jobs()][8]
  const uint32_t* jr;
  const uint32_t* gtab;
  const uint32_t* htab;
  const uint32_t* ext;    // [rows * lay.gparts()][24]
  uint32_t* proj;         // [rows * lay.jobs()][24]
  FbShape sh;             // always uniform in this build: sh.w bits in every window
  GpartLayout lay;
  ZK_HD void operator()(int t) const {
    const int row = t / lay.jobs(), g = lay.gpart_of_job(row, t % lay.jobs());
    uint32_t v[8], r[8];
    ld<8>(v, jv + (size_t)t * 8);
    ld<8>(r, jr + (size_t)t * 8);
    WarPt acc;
    // a value of 0 or 1: one table entry taken as (x : y : 1), or the identity
    if (g < 0 || scalar_le_one(v)) war_gpart(acc, gtab, v, sh.w);
    else war_ld_proj(acc, ext + ((size_t)row * lay.gparts() + g) * TOM_EXT_WORDS);
    war_accum_fixed(acc, htab, r, sh.w);
    war_st_proj(proj + (size_t)t * TOM_PROJ_WORDS, acc);
  }
};
