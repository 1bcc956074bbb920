// zkattest.cu — host orchestration + C ABI (include/zkattest.h) of libzkattest.
//
// One context = one CUDA device + one stream + a grow-only workspace.  A prove/verify call
// is a fixed sequence of ~25 batch kernels over flat arrays in HBM; there is no CPU compute
// path (the ZKA_HOSTSIM build of this file exists only for the CPU unit tests, see
// zk_launch.cuh).
#include "zkattest.h"

#include <math.h>
#include <stdio.h>

#include <algorithm>
#include <atomic>
#include <cmath>
#include <mutex>
#include <chrono>
#include <memory>
#include <thread>
#include <string>
#include <vector>

#include "zk_check.cuh"
#include "zk_launch.cuh"
#include "zk_prove.cuh"
#include "zk_seed.cuh"
#include "zk_trace.cuh"
#include "zk_verify_agg.cuh"
#if !defined(ZKA_HOSTSIM)
#include <cub/device/device_radix_sort.cuh>
#endif

namespace zk {
// ---- small helper tasks of the C ABI layer (namespace scope: kernel template arguments) ----
struct ParsePointsTask {   // host bytes -> affine Montgomery (+ validity), used for params / sub-ops
  const uint8_t* nist;   // [count][65] or null
  const uint8_t* tom;    // [count][67] or null
  uint32_t* nist_aff;    // [count][16]
  uint32_t* tom_aff;     // [count][18]
  uint8_t* bad;          // [count]
  uint8_t* inf;          // [count] (P-256 identity given as 65 zero bytes)
  ZK_HD void operator()(int t) const {
    if (nist) {
      P256Aff a;
      bool allz;
      const bool ok = p256_parse(a, allz, nist + (size_t)t * 65);
      if (!ok) p256_set_generator(a);
      p256_st_aff(nist_aff + (size_t)t * 16, a);
      if (bad) bad[t] = ok ? 0 : 1;
      if (inf) inf[t] = allz ? 1 : 0;
    }
    if (tom) {
      const uint8_t* b = tom + (size_t)t * WP;
      uint32_t xm[PGL], ym[PGL];
      bool ok = tom_parse(xm, ym, b);   // tag, coordinate range and curve equation (edwards.ts:70-86 / weier.ts:74-89)
      if (!ok) {
        TomPt g;
        tom_set_generator(g);
        copy_n<PGL>(xm, g.x);
        copy_n<PGL>(ym, g.y);
      }
      st<PGL>(tom_aff + (size_t)t * TOM_AFF_WORDS, xm);
      st<PGL>(tom_aff + (size_t)t * TOM_AFF_WORDS + PGL, ym);
      if (bad) bad[t] = ok ? 0 : 1;
    }
  }
};

struct GenAffTask {   // generator constants -> device
  uint32_t* p256_g;   // [16]
  uint32_t* tom_g;    // [18]
  ZK_HD void operator()(int) const {
    P256Aff g;
    p256_set_generator(g);
    p256_st_aff(p256_g, g);
    TomPt tg;
    tom_set_generator(tg);     // affine generator of the proof group (z = 1)
    st<PGL>(tom_g, tg.x);
    st<PGL>(tom_g + PGL, tg.y);
  }
};

template <class F, int NB>
struct FieldOpTask {
  const uint8_t *a, *b;
  uint8_t* out;
  int op;
  ZK_HD void operator()(int t) const {
    constexpr int N = F::N;
    uint32_t x[N], y[N], r[N];
    limbs_from_be<N>(x, a + (size_t)t * NB, NB);
    zero_n<N>(y);
    if (b) limbs_from_be<N>(y, b + (size_t)t * NB, NB);
    F::to_mont(x, x);
    F::to_mont(y, y);
    if (op == 0) F::mul(r, x, y);
    else if (op == 1) F::add(r, x, y);
    else if (op == 2) F::sub(r, x, y);
    else if (op == 3) F::inv(r, x);
    else F::inv_fermat(r, x);
    F::from_mont(r, r);
    limbs_to_be<N>(out + (size_t)t * NB, r, NB);
  }
};
struct GProjTask {
  const uint32_t* g;
  uint32_t* proj;
  ZK_HD void operator()(int) const {
    uint32_t one[PGL];
    PGp::set_one(one);
    st<PGL>(proj, g);
    st<PGL>(proj + PGL, g + PGL);
    st<PGL>(proj + 2 * PGL, one);
  }
};

struct CommitConvTask {
  const uint8_t *v, *r;
  uint32_t *jv, *jr;
  ZK_HD void operator()(int t) const {
    uint32_t a[8];
    limbs_from_be<8>(a, v + (size_t)t * 32, 32);
    reduce_once<FpP256>(a);
    st<8>(jv + (size_t)t * 8, a);
    limbs_from_be<8>(a, r + (size_t)t * 32, 32);
    reduce_once<FpP256>(a);
    st<8>(jr + (size_t)t * 8, a);
  }
};

struct PackTomTask {
  const uint8_t* bytes;
  uint8_t* out;
  ZK_HD void operator()(int t) const {
    for (int i = 0; i < WP; i++) out[(size_t)t * WP + i] = bytes[(size_t)t * BSTRIDE + i];
  }
};

struct P256MulTask {
  const uint8_t* k;
  const uint32_t* g8;
  const uint32_t* rtab;
  const uint8_t* binf;
  uint32_t* proj;
  ZK_HD void operator()(int t) const {
    uint32_t s[8];
    limbs_from_be<8>(s, k + (size_t)t * 32, 32);
    reduce_once<FnP256>(s);
    P256Pt acc;
    p256_set_identity(acc);
    if (rtab) {
      if (!binf[t]) p256_accum_rtab(acc, rtab + (size_t)t * RT_ENTRIES * P256_AFF_WORDS, s);
    } else {
      p256_accum_fixed(acc, g8, s, 8);
    }
    p256_st_proj(proj + (size_t)t * P256_PROJ_WORDS, acc);
  }
};

struct PackP256Task {
  const uint8_t* bytes;
  uint8_t* out;
  ZK_HD void operator()(int t) const {
    for (int i = 0; i < NP; i++) out[(size_t)t * NP + i] = bytes[(size_t)t * BSTRIDE + i];
  }
};

struct Hash80Task {
  const uint8_t* m;
  size_t stride;
  const uint32_t* len;
  uint8_t* out;
  ZK_HD void operator()(int t) const {
    Sha256 h;
    h.init();
    h.update(m + (size_t)t * stride, (int)len[t]);
    uint32_t c3[3];
    h.final80(c3);
    uint8_t* o = out + (size_t)t * 10;
    o[0] = (uint8_t)(c3[2] >> 8); o[1] = (uint8_t)c3[2];
    for (int i = 0; i < 4; i++) { o[2 + i] = (uint8_t)(c3[1] >> (24 - 8 * i)); o[6 + i] = (uint8_t)(c3[0] >> (24 - 8 * i)); }
  }
};

struct GenConvTask {
  const uint8_t* v;
  uint32_t *jv, *jr;
  ZK_HD void operator()(int) const {
    uint32_t a[8];
    limbs_from_be<8>(a, v, 32);
    reduce_once<FpP256>(a);
    st<8>(jv, a);
    zero_n<8>(a);
    st<8>(jr, a);
  }
};

struct KeyToIntTask {
  const uint32_t* aff;
  const uint8_t *bad, *inf;
  uint8_t* x;
  int32_t* status;
  ZK_HD void operator()(int t) const {
    uint32_t c[8];
    P256p::from_mont(c, aff + (size_t)t * 16);
    limbs_to_be<8>(x + (size_t)t * 32, c, 32);
    status[t] = (bad[t] || inf[t]) ? ZKA_ERR_INVALID_PK : ZKA_OK;
  }
};

// ---- multi-GPU helpers: proofs leave a rank as ONE contiguous block (zka_proofs_pack / zka_proofs_unpack)
ZK_HD uint64_t pack_align16(uint32_t len) { return ((uint64_t)len + 15u) & ~(uint64_t)15u; }
struct PackScanTask {   // off[b] = sum_{i<b} align16(len[i]); one thread (B <= a few thousand per group)
  const uint32_t* len;
  uint64_t* off;        // [B + 1]
  int B;
  ZK_HD void operator()(int) const {
    uint64_t acc = 0;
    for (int b = 0; b < B; b++) { off[b] = acc; acc += pack_align16(len[b]); }
    off[B] = acc;
  }
};
struct PackCopyTask {   // one thread per (proof, 16-byte piece); dir 0: rows -> packed, 1: packed -> rows
  uint8_t* rows;
  size_t stride;
  const uint32_t* len;
  const uint64_t* off;
  uint8_t* packed;
  size_t cap;
  int pieces;           // ceil(stride / 16)
  int dir;
  ZK_HD void operator()(int t) const {
    const int b = t / pieces, j = t % pieces;
    const size_t o = (size_t)16 * j;
    if (o >= len[b]) return;
    const size_t po = (size_t)off[b] + o;
    if (po + 16 > cap) return;   // the caller checks off[B] <= cap
    uint8_t* r = rows + (size_t)b * stride + o;
    uint8_t* q = packed + po;
    if (dir == 0) { for (int i = 0; i < 16; i++) q[i] = o + i < stride ? r[i] : 0; }
    else { for (int i = 0; i < 16; i++) if (o + i < stride) r[i] = q[i]; }
  }
};
struct PackCopy16Task {   // same, both sides 16-byte aligned: one uint4 per thread
  uint8_t* rows;
  size_t stride;
  const uint32_t* len;
  const uint64_t* off;
  uint8_t* packed;
  size_t cap;
  int pieces;
  int dir;
  ZK_HD void operator()(int t) const {
    const int b = t / pieces, j = t % pieces;
    const size_t o = (size_t)16 * j;
    if (o >= len[b]) return;
    const size_t po = (size_t)off[b] + o;
    if (po + 16 > cap) return;
    U4* r = reinterpret_cast<U4*>(rows + (size_t)b * stride + o);
    U4* q = reinterpret_cast<U4*>(packed + po);
    if (dir == 0) *q = *r; else *r = *q;
  }
};

}  // namespace zk

using namespace zk;

namespace {

struct FixedTable {   // positional table of one base point
  DevBuf buf;
  uint32_t* tab = nullptr;
};

}  // namespace

// A lane = one compute stream + two copy streams + its own grow-only workspace.  A prove / verify call cuts
// the batch into chunks and deals them round-robin to the lanes; every lane beyond the first is driven by
// its own host thread for the duration of the call, so the mid-pipeline host synchronisation of one lane
// (the item count after the Fiat-Shamir scan) never stalls the others, the latency-bound stages of one
// chunk (doubling chains, 16 KB hashes, scans) overlap the multiplier-bound kernels of another, and
// host<->device copies of one lane overlap the kernels of the others.
struct Lane {
  Stream st;
  // copy streams + events of the host-buffer pipeline; slot = (lane-local chunk index) & 1
  Stream cs_in, cs_out;
  Event ev_small[2], ev_tape[2], ev_done[2], ev_out[2];
  Stream aux[2];            // verifier: the torsion guard and the P-256 part of the aggregate check run beside the tomEdwards256 MSM
  Event ev_fork, ev_join[2];
  // workspace (grow-only pools, see Cursor): one chunk pass, the input and output staging buffers of each slot, and the
  // verifier's chunk-wide aggregate check (zk_verify_agg.cuh: its fixed parts, and one pool per MSM as the two MSMs
  // run side by side)
  DevBuf w[52];
  DevBuf in[2][10], out[2][3];
  DevBuf agg[9], agg_tom[5 + 2 * AGG_MAX_LEVELS], agg_nist[5 + 2 * AGG_MAX_LEVELS];
  // the prover's self-check (check_chunk): c_b, the rows to check, the verify tape, ok and the verifier's statuses; and the
  // lane's counts of rows checked / failed over one call
  DevBuf chk[5], chk_count;
  std::string err;
  ~Lane() {
    for (int i = 0; i < 2; i++) {
      ev_destroy(ev_small[i]); ev_destroy(ev_tape[i]); ev_destroy(ev_done[i]); ev_destroy(ev_out[i]);
    }
    ev_destroy(ev_fork); ev_destroy(ev_join[0]); ev_destroy(ev_join[1]);
    stream_destroy(cs_in);
    stream_destroy(cs_out);
    stream_destroy(aux[0]);
    stream_destroy(aux[1]);
    stream_destroy(st);
  }
};

struct zka_ctx : Lane {
  int device = 0;
  std::vector<std::unique_ptr<Lane>> extra;   // lanes 1 .. nlanes-1 (lane 0 is the context itself)
  int nlanes = 3;             // ZKA_LANES
  DevBuf ring_in, ring_m;     // the ring of the current call (shared by all lanes, read-only while they run)
  DevBuf ring_leaves, ring_digest;   // its hedge digest (RingDigestTask) when the call is hedged
  Lane& lane(int i) { return i == 0 ? *this : *extra[i - 1]; }
#if defined(ZKA_PG_WAR256)
  FbShape tom = fb_uniform(22);   // shape of the proof group's fixed-base tables g and h (ZKA_TOM_W)
#else
  FbShape tom = fb_lookups(11);   // 7 windows of 23 bits + 4 of 24: 7 (2^22 + 1) + 4 (2^23 + 1) signed-digit entries x 128 B =
                                  // 8.05 GB of HBM per base (ZKA_TOM_NWIN, ZKA_TOM_W)
#endif
  size_t tom_table_max = 0;       // a proof-group table above this many bytes counts as an allocation that failed (ZKA_TOM_TABLE_MAX)
  bool tom_fallback = false;      // the tables of the shape asked for did not fit: this context walks one lookup more (zka_stat)
  int chunk = 4096;       // largest chunk of a call whose buffers are all device memory (ZKA_CHUNK)
  int host_chunk = 2048;  // chunk size when proofs return to host memory: copies of one chunk overlap the next
  volatile uint32_t* progress = nullptr;   // zka_set_progress: flags[k] = 1 when chunk k of the running prove call is complete
  uint32_t progress_cap = 0;
  int agg = 1;            // verifier: chunk-wide aggregate check before the per-proof MSMs (ZKA_AGG=0 disables it)
  int agg_c = 0;          // window bits of the aggregate MSM (0: chosen from the chunk size; ZKA_AGG_C)
  uint64_t agg_pass = 0, agg_fail = 0;   // chunks decided by the aggregate / sent to the per-proof path (zka_stat)
  int self_check = 0;     // prover: verify every proof with samples = sec_level before releasing it (check_chunk)
  uint64_t self_check_rows = 0, self_check_fail = 0;   // rows checked / given ZKA_ERR_SELF_CHECK (zka_stat)
  std::mutex stat_mu;
  std::mutex copy_mu;     // keeps the copies of one chunk together on the shared copy-in stream (verify)
  int agg_c_last = 0;
  bool tape_split = true; // host tapes travel in two strided copies: the 3 + 4S draws before the challenge, then only the
                          // item / GK draws up to the longest proof of the chunk (ZKA_TAPE_SPLIT=0: one full-stride copy)
  int p256_hw = 20;       // window bits of the P-256 G table and of the per-params NistGroup.h table
                          // (13 windows x 2^20 entries x 64 B = 872 MB each)
  FixedTable g8;          // P-256 generator, w=8 [32][256][16]
  FixedTable gw;          // P-256 generator, p256_hw-bit windows (prover phase A)
  FixedTable tg;          // tomEdwards256 generator [nwin][2^w][32]
  DevBuf tg_bytes;        // 67-byte encoding of g
  DevBuf lag;             // GK Lagrange matrix cache
  int lag_n = -1;
  DevBuf trace[32];       // workspace of the trace stages (zk_trace.cuh), which run after the untraced passes
};

struct zka_params {
  zka_ctx* ctx = nullptr;
  uint32_t sec_level = 80;
  FixedTable h8;          // NistGroup.h fixed-base table, h_w-bit windows (16 x 65536 x 64 B = 67 MB)
  int h_w = 20;
  FixedTable th;          // ProofGroup.h table
  uint8_t h_nist[65];
  uint8_t h_proof[WP];
  uint8_t hedge_digest[32];   // the params digest of the hedged seeds (include/zkattest.h)
};

// R rings on the device (zka_rings_create): ring r is reduced mod the proof-group order and padded to 2^n_r entries with
// its own first entry, at entry ring_base[r] of ring_m
struct zka_rings {
  zka_ctx* ctx = nullptr;
  uint32_t R = 0;
  std::vector<uint32_t> size;              // N_r
  std::vector<int> depth;                  // n_r = ceil(log2 N_r)
  DevBuf ring_m, ring_base, ring_size, ring_depth;   // [total][8], [R], [R], [R]
  DevBuf lag;                              // the prover's GK Lagrange matrices of the depths 1 .. max n_r (GkLagrangeSetTask)
  DevBuf ring_digest;                      // [R][32] the hedge digest of each ring (RingDigestTask)
};

namespace {

int fail(zka_ctx* ctx, int code, const std::string& msg) {
  if (ctx) ctx->err = msg;
  return code;
}
// runs the body of an entry point: an exception (a CUDA error) becomes ZKA_E_CUDA with its message
template <class Fn>
int guarded(zka_ctx* ctx, Fn&& body) {
  try {
    return body();
  } catch (const std::exception& e) {
    return fail(ctx, ZKA_E_CUDA, e.what());
  }
}

// ---- chunk-wide aggregate check of the verifier (zk_verify_agg.cuh; the plan is agg_plan there) -------------------
// enqueue histogram, prefix sums, scatter, bucket sums and the reduction tree of one group; returns the root sums
template <class Src>
void agg_msm(Stream& st, Cursor A, const Src& src, const AggPlan& pl, const uint32_t* ctl, const uint32_t** rootA,
             const uint32_t** rootB) {
  const AggDigits& D = pl.D;
  const int nwin = D.nwin, nb = D.nb, nseg = (nb + 1 + AGG_SEG - 1) / AGG_SEG;
  const size_t cap = (size_t)src.slots();
  uint32_t* hist = A.take<uint32_t>((size_t)nwin * (nb + 1));
  uint32_t* bstart = A.take<uint32_t>((size_t)nwin * (nb + 2));
  uint32_t* segtot = A.take<uint32_t>((size_t)nwin * nseg);
  uint32_t* sorted = A.take<uint32_t>((size_t)nwin * cap);
  uint32_t* bsum = A.take<uint32_t>((size_t)nwin * nb * Src::PTW);
  dev_memset(st, hist, 0, (size_t)nwin * (nb + 1) * 4);
  launch(st, (long long)cap, AggHistTask<Src>{src, D, ctl, hist});
  launch(st, (long long)nwin * nseg, AggSegSumTask{ctl, hist, segtot, nb, nseg});
  launch(st, nwin, AggSegScanTask{ctl, segtot, nseg});
  launch(st, (long long)nwin * nseg, AggOffsetsTask{ctl, segtot, hist, bstart, nb, nseg});
  launch(st, (long long)cap, AggScatterTask<Src>{src, D, ctl, hist, sorted, cap});
  launch(st, (long long)nwin * nb, AggBucketTask<Src>{src, ctl, bstart, sorted, bsum, cap, nb});
  const uint32_t *inA = bsum, *inB = nullptr;
  int nin = nb, ll = 0;
  for (int lv = 0; lv < pl.levels; lv++) {
    const int nout = nin >> pl.lm[lv];
    uint32_t* oA = A.take<uint32_t>((size_t)nwin * nout * Src::PTW);
    uint32_t* oB = A.take<uint32_t>((size_t)nwin * nout * Src::PTW);
    launch(st, (long long)nwin * nout, AggLevelTask<Src>{ctl, inA, inB, oA, oB, nin, pl.lm[lv], ll, nwin, D.top_shift});
    inA = oA; inB = oB; nin = nout; ll += pl.lm[lv];
  }
  *rootA = inA;
  *rootB = inB;
}

int ceil_log2(uint32_t v) {
  int n = 0;
  while ((1ull << n) < v) n++;
  return n;
}


// Normalisation launches: points per thread (= per binary inversion).  A thread costs about
// per_point * chunk + 70 multiplications in sequence (the inversion is worth ~70), and the grid runs in
// waves of (SMs x 4 resident CTAs): pick the chunk that minimises waves x thread length.  (The first
// heuristic, count / 100000, put 1.4 waves on the GPU for a 1024-proof batch.)
static int g_norm_slots = 132 * 4;   // SMs x 4, read from the device in zka_init
static bool g_norm_model = true;
inline int norm_chunk_for(long long count, int per_point = 11) {
  if (!g_norm_model) {
    long long c = count / 100000;
    if (c < 8) c = 8;
    if (c > NORM_CHUNK_MAX) c = NORM_CHUNK_MAX;
    return (int)c;
  }
  int best = 8;
  long long best_cost = -1;
  for (int c = 8; c <= NORM_CHUNK_MAX; c++) {
    const long long threads = (count + c - 1) / c, ctas = (threads + 127) / 128;
    const long long waves = (ctas + g_norm_slots - 1) / g_norm_slots;
    const long long cost = waves * ((long long)per_point * c + 70);
    if (best_cost < 0 || cost < best_cost) { best_cost = cost; best = c; }
  }
  return best;
}
inline void launch_p256_norm(Stream& st, const uint32_t* proj, uint32_t* aff, uint8_t* bytes, uint8_t* inf, long long count) {
  if (count <= 0) return;
  const int ch = norm_chunk_for(count, bytes ? 7 : 5);
  launch(st, (count + ch - 1) / ch, P256NormTask{proj, aff, bytes, inf, (int)count, ch});
}
// e2 = 1: the points come from TomCommitTask / TomCommitHTask (E, F, G, H on the a = -1 image curve E2, TOM_E2_WORDS
// apart); e2 = 0: E1 projective (X, Y, Z), TOM_PROJ_WORDS apart unless `stride` says otherwise
// aff may be null; otherwise the E1 affine pair is written for points with (index % aff_mod) < aff_lim
inline void launch_tom_norm(Stream& st, const uint32_t* proj, uint32_t* aff, uint8_t* bytes, long long count, int e2,
                            int aff_mod = 1, int aff_lim = 1, int stride = 0) {
  if (count <= 0) return;
  const int ch = norm_chunk_for(count);
  if (stride == 0) stride = e2 ? TOM_E2_WORDS : TOM_PROJ_WORDS;
  launch(st, (count + ch - 1) / ch, TomNormTask{proj, aff, bytes, (int)count, ch, e2, aff_mod, aff_lim, stride});
}

// ---- table construction -------------------------------------------------------------------
// P-256 positional table (signed digits, fb_entries(w) multiples per window) from one affine Montgomery base
// (device pointer, 16 words)
void build_p256_tab(zka_ctx* ctx, const uint32_t* base_aff_dev, FixedTable& out, int w) {
  Stream& st = ctx->st;
  const int nwin = fb_windows(w);
  const size_t E = (size_t)fb_entries(w), count = (size_t)nwin * E;
  DevBuf pows, rows;
  uint32_t* d_pows = pows.get<uint32_t>((size_t)nwin * P256_PROJ_WORDS);
  uint32_t* d_rows = rows.get<uint32_t>(count * P256_PROJ_WORDS);
  out.tab = out.buf.get<uint32_t>(count * P256_AFF_WORDS);
  launch(st, 1, P256PowsTask{base_aff_dev, nullptr, d_pows, 1, nwin, w});
  if (w > 9) {
    DevBuf hi;
    const int nh = 1 << (w - 9);
    uint32_t* d_hi = hi.get<uint32_t>((size_t)nwin * nh * P256_PROJ_WORDS);
    launch(st, nwin, P256RowsHiTask{d_pows, d_hi, d_rows, w});
    launch(st, (long long)nwin * nh, P256RowsLoTask{d_pows, d_hi, d_rows, w});
    sync(st);   // hi is freed at the end of this block, before the normalisation
  } else {
    launch(st, nwin, P256RowsTask{d_pows, d_rows, w});
  }
  launch_p256_norm(st, d_rows, out.tab, nullptr, nullptr, (long long)(count));
  sync(st);
}
// memory of one proof-group table of shape ctx->tom; throws when it exceeds ZKA_TOM_TABLE_MAX or the device has no room
uint32_t* alloc_tom_tab(zka_ctx* ctx, DevBuf& buf) {
  const size_t words = ctx->tom.total() * TOM_PRE_WORDS;
  if (ctx->tom_table_max && words * sizeof(uint32_t) > ctx->tom_table_max)
    throw std::runtime_error("proof-group fixed-base table of " + std::to_string(words * sizeof(uint32_t)) + " bytes exceeds ZKA_TOM_TABLE_MAX");
  return buf.get_exact<uint32_t>(words);
}
#if defined(ZKA_PG_WAR256)
// war256 positional table [fb_windows(w)][fb_entries(w)] of affine points from one affine base (16 words, device)
void build_tom_tab(zka_ctx* ctx, const uint32_t* base_aff_dev, FixedTable& out) {
  Stream& st = ctx->st;
  const int w = ctx->tom.w, nwin = ctx->tom.nwin;
  const size_t E = (size_t)fb_entries(w), count = (size_t)nwin * E;
  DevBuf pows, rows;
  uint32_t* d_pows = pows.get<uint32_t>((size_t)nwin * P256_PROJ_WORDS);
  uint32_t* d_rows = rows.get<uint32_t>(count * P256_PROJ_WORDS);
  out.tab = alloc_tom_tab(ctx, out.buf);
  launch(st, 1, WarPowsTask{base_aff_dev, nullptr, d_pows, 1, nwin, w});
  if (w > 9) {
    DevBuf hi;
    const int nh = 1 << (w - 9);
    uint32_t* d_hi = hi.get<uint32_t>((size_t)nwin * nh * P256_PROJ_WORDS);
    launch(st, nwin, WarRowsHiTask{d_pows, d_hi, d_rows, w});
    launch(st, (long long)nwin * nh, WarRowsLoTask{d_pows, d_hi, d_rows, w});
    sync(st);   // hi is freed at the end of this block, before the normalisation
  } else {
    launch(st, nwin, WarRowsTask{d_pows, d_rows, w});
  }
  {
    const int ch = norm_chunk_for((long long)count, 5);
    launch(st, ((long long)count + ch - 1) / ch, WarNormTask{d_rows, out.tab, nullptr, nullptr, (int)count, ch});
  }
  sync(st);
}
#else
// tomEdwards256 positional table of shape ctx->tom from one image-curve affine base (18 words, device).  Built window
// by window through one staging buffer of projective rows, which is therefore as large as the widest window (0.94 GB
// at 24 bits) and not as the table.
void build_tom_tab(zka_ctx* ctx, const uint32_t* base_aff_dev, FixedTable& out) {
  Stream& st = ctx->st;
  const FbShape sh = ctx->tom;
  out.tab = alloc_tom_tab(ctx, out.buf);
  DevBuf pows, rows, hi;
  uint32_t* d_pows = pows.get<uint32_t>((size_t)sh.nwin * 36);
  uint32_t* d_rows = rows.get<uint32_t>(sh.entries(sh.nwin - 1) * TOM_PROJ_WORDS);
  launch(st, 1, TomPowsTask{base_aff_dev, d_pows, 1, sh});
  const bool two_level = sh.w > 9;
  uint32_t* d_hi = nullptr;
  if (two_level) {
    d_hi = hi.get<uint32_t>(tom_hi_offset(sh, sh.nwin) * 36);
    launch(st, sh.nwin, TomRowsHiTask{d_pows, d_hi, sh});
  }
  for (int j = 0; j < sh.nwin; j++) {
    const size_t ne = sh.entries(j);
    const uint32_t* pw = d_pows + (size_t)j * 36;
    if (two_level) {
      const int nh = 1 << (sh.width(j) - 9);
      launch(st, nh + 1, TomRowsLoTask{pw, d_hi + tom_hi_offset(sh, j) * 36, d_rows, nh});
    } else {
      launch(st, 1, TomRowsTask{pw, d_rows, sh.width(j)});
    }
    // rows (E1 projective) -> entries of the prover's a = -1 image curve (v - w, v + w, 2 d2 w v)
    launch(st, (long long)(ne + 15) / 16, TomTabE2Task{d_rows, out.tab + sh.offset(j) * TOM_PRE_WORDS, (int)ne});
  }
  sync(st);
}

#endif

// stage a caller buffer on the device if it is a host pointer
template <class T>
const T* stage_in(Stream& st, DevBuf& buf, const T* p, size_t count) {
  if (!p || count == 0) return p;
  if (is_device_ptr(p)) return p;
  T* d = buf.get<T>(count);
  copy_h2d(st, d, p, count * sizeof(T));
  return d;
}

// A caller output of `width` T per row.  Kernels write rows [b0, b0 + rows) in place when it is device memory, otherwise
// into a staging buffer that copy_back then queues for the caller.
template <class T>
struct Output {
  T* dst;
  size_t width;
  bool dev;
  Output(T* p, size_t width) : dst(p), width(width), dev(is_device_ptr(p)) {}
  T* rows(DevBuf& stage, uint32_t b0, size_t rows) const { return dev ? dst + b0 * width : stage.get<T>(rows * width); }
  void copy_back(Stream& st, uint32_t b0, const T* d, size_t rows) const {
    if (!dev) copy_d2h(st, dst + b0 * width, d, rows * width * sizeof(T));
  }
  // only the first `bytes` of each row
  void copy_back_2d(Stream& st, uint32_t b0, const T* d, size_t rows, size_t bytes) const {
    if (!dev) copy_d2h_2d(st, dst + b0 * width, width * sizeof(T), d, width * sizeof(T), bytes, rows);
  }
};

// Chunk schedule of a call: boundaries off[0..nchunks] of the batch.  `cmax` = largest chunk, `lanes` = lanes that
// will run.  Plain: near-equal chunks, at least one per lane when chunks of >= 256 proofs allow it.  Tapered (used
// when a buffer lives in host memory): the first chunks are small so that the kernels start after a short input
// copy, the last ones small so that little output copy is left exposed after the last kernel, and lanes that
// claim chunks dynamically drift out of phase (one copies while another computes):
//   cmax/4, cmax/2, [full chunks], cmax/2, cmax/4.
std::vector<uint32_t> chunk_schedule(uint32_t B, uint32_t cmax, int lanes, bool taper) {
  std::vector<uint32_t> off{0};
  auto r32 = [](uint32_t v) { return v < 32 ? std::max<uint32_t>(v, 1) : ((v + 31) & ~31u); };
  if (lanes > 1) {
    uint32_t per = r32((B + (uint32_t)lanes - 1) / (uint32_t)lanes);
    cmax = std::min(cmax, std::max<uint32_t>(per, 256));
  }
  uint32_t done = 0;
  auto push = [&](uint32_t n) { n = std::min(n, B - done); if (n) { done += n; off.push_back(done); } };
  if (taper && cmax >= 1024 && B >= 3 * cmax) {
    const uint32_t q = r32(cmax / 4), h = r32(cmax / 2);
    push(q);
    push(h);
    const uint32_t mid = B - done - (h + q);
    const uint32_t nm = (mid + cmax - 1) / cmax;
    const uint32_t each = r32((mid + nm - 1) / nm);
    for (uint32_t i = 0; i + 1 < nm; i++) push(each);
    push(B - done - (h + q));
    push(h);
    push(q);
  } else {
    const uint32_t nk = (B + cmax - 1) / cmax;
    const uint32_t each = r32((B + nk - 1) / nk);
    while (done < B) push(each);
  }
  return off;
}

// flags[k] = 1 once everything enqueued on `st` so far has run (a CUDA host callback: no thread of ours waits)
#if !defined(ZKA_HOSTSIM)
void CUDART_CB progress_cb(void* p) { *reinterpret_cast<volatile uint32_t*>(p) = 1u; }
void notify_progress(Stream& st, volatile uint32_t* flag) { ZK_CUDA_CHECK(cudaLaunchHostFunc(st.s, progress_cb, (void*)flag)); }
#else
void notify_progress(Stream&, volatile uint32_t* flag) { *flag = 1u; }
#endif

// Run fn(lane index) for lanes 0..used-1: lane 0 on the calling thread, the others on their own host threads
// (each binds the context's device).  The first exception of any lane is rethrown on the caller.
template <class Fn>
void run_lanes(zka_ctx* ctx, int used, Fn fn) {
  if (used <= 1) { fn(0); return; }
  std::vector<std::thread> th;
  std::vector<std::exception_ptr> errs((size_t)used);
  for (int li = 1; li < used; li++)
    th.emplace_back([&, li] {
      try {
#if !defined(ZKA_HOSTSIM)
        ZK_CUDA_CHECK(cudaSetDevice(ctx->device));
#endif
        fn(li);
      } catch (...) {
        errs[(size_t)li] = std::current_exception();
      }
    });
  try { fn(0); } catch (...) { errs[0] = std::current_exception(); }
  for (auto& t : th) t.join();
  for (auto& e : errs)
    if (e) std::rethrow_exception(e);
}

// ---- stage chains shared by the batched pipelines and the stand-alone sub-proof paths
// The GK Lagrange matrix of the prover: it depends only on n and is cached per context
void prep_lagrange(zka_ctx* ctx, Stream& st, int n) {
  if (ctx->lag_n != n) {
    launch(st, 1, GkLagrangeTask{ctx->lag.get<uint32_t>((size_t)n * n * 8), n});
    ctx->lag_n = n;
  }
}
// The ring of a call on the device (RingPrepTask), for the prover the Lagrange matrix, and for a hedged call the ring's
// digest into ctx->ring_digest (RingDigestTask: leaves, then root).
const uint32_t* prep_ring(zka_ctx* ctx, Stream& st, const uint8_t* ring, uint32_t N, int n, bool lagrange, bool digest = false) {
  const uint8_t* d_ring = stage_in(st, ctx->ring_in, ring, (size_t)N * 32);
  uint32_t* ring_m = ctx->ring_m.get<uint32_t>(((size_t)1 << n) * 8);
  launch(st, 1ll << n, RingPrepTask{d_ring, ring_m, (int)N});
  if (lagrange) prep_lagrange(ctx, st, n);
  if (digest) {
    const uint32_t nl = hedge_leaves(n);
    RingDigestTask t{ring_m, nullptr, nullptr, nullptr, nullptr, N, (uint32_t)n, 1u, ctx->ring_leaves.get<uint8_t>((size_t)32 * nl),
                     ctx->ring_digest.get<uint8_t>(32), false};
    launch(st, nl, t);
    t.root = true;
    launch(st, 1, t);
  }
  return ring_m;
}

// The per-row arguments of a batched prove call (host or device), exactly one of tape / seeds set, or hedge (seeds then
// optional: each row's seed is derived from them, the statement and the signature, SeedHedgeTask).  proveExp alone reads
// base / s_in / q_in instead of msg_hash / sig / which; ring_of is set for a ring-set call.
struct ProveRows {
  const uint8_t *msg_hash{}, *sig{}, *pk{}, *base{}, *s_in{}, *q_in{}, *tape{}, *seeds{};
  const uint32_t *which{}, *ring_of{};
  size_t tape_stride{}, proof_stride{};
  uint8_t* proofs{}; uint32_t* proof_len{}; int32_t* status{};
  bool hedge = false;
  ProveRows() = default;
  ProveRows(uint8_t* proofs, size_t stride, uint32_t* len, int32_t* status) : proof_stride(stride), proofs(proofs), proof_len(len), status(status) {}
  // the rows from r0 on, null pointers left null (the one place that knows each row's width)
  ProveRows at(size_t r0) const {
    ProveRows v = *this;
    auto skip = [r0](auto*& p, size_t width) { if (p) p += r0 * width; };
    skip(v.msg_hash, 32); skip(v.sig, 64); skip(v.pk, 65); skip(v.which, 1); skip(v.ring_of, 1); skip(v.base, 65);
    skip(v.s_in, 32); skip(v.q_in, 65); skip(v.seeds, 32); skip(v.tape, tape_stride);
    skip(v.proofs, proof_stride); skip(v.proof_len, 1); skip(v.status, 1);
    return v;
  }
};
// The same for a batched verify call; q_ext (verifyExp alone, device memory) holds each row's Q
struct VerifyRows {
  const uint8_t *msg_hash{}, *proofs{}, *tape{}, *seeds{}, *q_ext{};
  const uint32_t *proof_len{}, *ring_of{};
  size_t proof_stride{}, tape_stride{};
  uint8_t* ok{}; int32_t* status{};
  VerifyRows() = default;
  VerifyRows(const uint8_t* proofs, size_t stride, const uint32_t* len, uint8_t* ok, int32_t* status)
      : proofs(proofs), proof_len(len), proof_stride(stride), ok(ok), status(status) {}
  VerifyRows at(size_t r0) const {
    VerifyRows v = *this;
    auto skip = [r0](auto*& p, size_t width) { if (p) p += r0 * width; };
    skip(v.msg_hash, 32); skip(v.proofs, proof_stride); skip(v.proof_len, 1); skip(v.tape, tape_stride); skip(v.seeds, 32);
    skip(v.ring_of, 1); skip(v.q_ext, NP); skip(v.ok, 1); skip(v.status, 1);
    return v;
  }
};

// Where the rows of a batched call find their ring: one ring of N keys for every row, or a set, whose rows (ring_of) each
// have the ring and the depth of their own; n, the depth the chunks are laid out for, is then the largest depth the rows
// use (a set call enters ring_passes as pass(set, 0)).  proveExp / verifyExp alone have neither and keep N = 2.
struct RingSrc {
  const uint8_t* ring; uint32_t N;   // one ring, or
  const zka_rings* set; int n;       // a set
  static RingSrc one(const uint8_t* ring, uint32_t N) { return {ring, N, nullptr, ceil_log2(N)}; }
  static RingSrc pass(const zka_rings* set, int n) { return {nullptr, 0, set, n}; }
  static RingSrc none(int n) { return {nullptr, 2, nullptr, n}; }
  // the call's ring on the device, for the prover the Lagrange matrix and for a hedged call the ring digest: once per
  // call, done before the lanes start
  const uint32_t* prepare(zka_ctx* ctx, bool lagrange, bool digest = false) const {
    if (!set && !ring) return nullptr;
    if (set) return (const uint32_t*)set->ring_m.p;   // prepared by zka_rings_create, with the matrices and digests
    const uint32_t* ring_m = prep_ring(ctx, ctx->st, ring, N, n, lagrange, digest);
    sync(ctx->st);
    return ring_m;
  }
  // [R][32] ring digests (one ring: R = 1), after prepare(.., digest = true)
  const uint8_t* digests(const zka_ctx* ctx) const { return (const uint8_t*)(set ? set->ring_digest.p : ctx->ring_digest.p); }
  // a chunk's ring fields; ring_of: the chunk's rows of it on the device
  template <class Ctx>
  void fill(Ctx& c, const uint32_t* ring_m, const uint32_t* ring_of) const {
    c.ring_m = ring_m;
    if (!set) return;
    c.ring_of = ring_of;
    c.ring_base = (const uint32_t*)set->ring_base.p;
    c.ring_depth = (const uint32_t*)set->ring_depth.p;
    if constexpr (std::is_same<Ctx, ProveCtx>::value) {
      c.ring_size = (const uint32_t*)set->ring_size.p;
      c.gk_lag = (uint32_t*)set->lag.p;
    }
  }
};

// A batched call after its null checks: its ring's checks, check(largest depth used), then ONE pass(ring) over all B rows.
// For a set the chunks' launch geometry (B n GK threads, 4n + 1 GK scalars per proof, the tape row widths) takes the largest
// depth the rows use and every row follows its own (n_row), whatever the order of depths in ring_of.  A set's ring_of is
// read on the host (4 bytes per row, copied when it is device memory) to check the indices and find that depth.
template <class Check, class Pass>
int ring_passes(zka_ctx* ctx, const RingSrc& ring, const uint32_t* ring_of, uint32_t B, Check check, Pass pass) {
  if (ring.set && ring.set->ctx != ctx) return fail(ctx, ZKA_E_ARG, "ring set of another context");
  if (B == 0) return 0;
  return guarded(ctx, [&] {
    if (!ring.set) {
      // N = 1 makes hashPoints([]) throw in the reference (group.ts:223 reduce of an empty array)
      if (ring.N < 2 || ring.N > (1u << 20)) return fail(ctx, ZKA_E_ARG, "ring size must be in [2, 2^20]");
      const int rc = check(ring.n);
      return rc ? rc : pass(ring);
    }
    std::vector<uint32_t> h(B);
    if (is_device_ptr(ring_of)) {
      copy_d2h(ctx->st, h.data(), ring_of, (size_t)B * 4);
      sync(ctx->st);
    } else {
      memcpy(h.data(), ring_of, (size_t)B * 4);
    }
    const std::vector<int>& depth = ring.set->depth;
    int nmax = 0;
    for (uint32_t b = 0; b < B; b++) {
      if (h[b] >= ring.set->R) return fail(ctx, ZKA_E_ARG, "ring_of[i] >= number of rings in the set");
      nmax = std::max(nmax, depth[h[b]]);
    }
    const int rc = check(nmax);
    return rc ? rc : pass(RingSrc::pass(ring.set, nmax));
  });
}

int gk_blocks(int n) { return 1 << (n - gk_block_bits(n)); }   // ring blocks of the GK polynomial kernels

// the fields every prover shares: dimensions, tables, window bits
ProveCtx prove_ctx(const zka_ctx* ctx, const zka_params* P, int B, int S, int N, int n) {
  ProveCtx c;
  memset(&c, 0, sizeof(c));
  c.B = B; c.S = S; c.N = N; c.n = n;
  c.tom = ctx->tom;
  c.g_tab8 = ctx->g8.tab; c.h_tab8 = P->h8.tab; c.h_w = P->h_w;
  c.g_tabw = ctx->gw.tab; c.g_w = ctx->p256_hw;
  c.tg_tab = ctx->tg.tab; c.th_tab = P->th.tab;
  c.tg_bytes = (const uint8_t*)ctx->tg_bytes.p;
  c.gk_lag = (uint32_t*)ctx->lag.p;
  return c;
}
// the same for every verifier
VerifyCtx verify_ctx(const zka_ctx* ctx, const zka_params* P, int B, int S, int N, int n, int K, int mode) {
  VerifyCtx c;
  memset(&c, 0, sizeof(c));
  c.B = B; c.S = S; c.N = N; c.n = n; c.K = K; c.mode = mode;
  c.tom = ctx->tom;
  c.g_tab8 = ctx->g8.tab; c.h_tab8 = P->h8.tab; c.h_w = P->h_w;
  c.tg_tab = ctx->tg.tab; c.th_tab = P->th.tab;
  c.tg_bytes = (const uint8_t*)ctx->tg_bytes.p;
  return c;
}

// commitments of the first store: pkX, pkY and Tx, Ty of every repetition
void prove_store1(Stream& st, const ProveCtx& c) {
  const long long n1 = (long long)c.B * (2 + 2 * c.S);
  launch(st, n1, JobsATask{c});
  launch(st, n1, TomCommitTask{c.s1_jv, c.s1_jr, c.tg_tab, c.th_tab, c.s1_proj, c.tom});
  launch_tom_norm(st, c.s1_proj, c.s1_aff, c.s1_bytes, n1, 1);
}
// The c.M items of the 0-bit repetitions (pointAdd.ts:92-163 each), from their secrets to their bytes in the proof rows,
// and the Groth-Kohlweiss commitments of the membership proof (gk.ts:129-176) with their encodings, behind the items in
// the s2 arrays.  The stages of the two alternate (with host buffers the batched prover was measurably slower with one
// chain after the other); provePointAdd alone runs only the items, proveMembership alone only the GK part.  gext:
// prove_gext_words(c) words for the g-parts of the commitments (GpartLayout), [M][GJOBS_PER_ITEM] of the items and
// behind them [B][2n] of the GK rows; c.gk_part: the block sums when the ring is cut into blocks.
size_t prove_gext_words(const ProveCtx& c) { return ((size_t)c.M * GJOBS_PER_ITEM + (size_t)c.B * 2 * c.n) * TOM_EXT_WORDS; }
void prove_items_gk(Stream& st, const ProveCtx& c, uint32_t* gext, bool items, bool gk) {
  const long long M = c.M, nj = M * JOBS_PER_ITEM, nd = M * DERS_PER_ITEM;
  const long long Bn = (long long)c.B * c.n, ng = 4 * Bn;
  const int nblk = gk_blocks(c.n);
  const size_t g0 = c.s2_gk(0, 0);
  const GpartLayout item_lay{0, nullptr, nullptr}, gk_lay{c.n, c.ring_of, c.ring_depth};
  uint32_t* gk_ext = gext + (size_t)M * GJOBS_PER_ITEM * TOM_EXT_WORDS;
  if (items) {
    launch(st, (M + ITEM_INV_CHUNK - 1) / ITEM_INV_CHUNK, ItemInvTask{c});
    launch(st, M, ItemScalarsTask{c});
  }
  if (gk) {
    launch(st, Bn, GkJobsTask{c});
    launch(st, Bn * nblk, GkPolyTask{c});
    if (nblk > 1) launch(st, Bn, GkPolyReduceTask{c});
    launch(st, Bn, GkCdJobsTask{c});
  }
  if (items) {   // item jobs: g-parts once per distinct committed value, then r*h on top (TomCommitG/HTask)
    launch(st, M * GJOBS_PER_ITEM, TomCommitGTask{c.s2_jv, c.tg_tab, gext, c.tom, item_lay});
    launch(st, nj, TomCommitHTask{c.s2_jv, c.s2_jr, c.tg_tab, c.th_tab, gext, c.s2_proj, c.tom, item_lay});
  }
  if (gk) {      // GK jobs: g-parts of ca_i and cd_i only
    launch(st, 2 * Bn, TomCommitGTask{c.s2_jv + g0 * 8, c.tg_tab, gk_ext, c.tom, gk_lay});
    launch(st, ng, TomCommitHTask{c.s2_jv + g0 * 8, c.s2_jr + g0 * 8, c.tg_tab, c.th_tab, gk_ext, c.s2_proj + g0 * TOM_E2_WORDS,
                                  c.tom, gk_lay});
  }
  if (items) {
    // only T1x, T1y (jobs 0, 1 of each item) are needed again as points (DerivedTask)
    launch_tom_norm(st, c.s2_proj, c.s2_aff, c.s2_bytes, nj, 1, JOBS_PER_ITEM, 2);
    launch(st, M, DerivedTask{c});
    // derived points come from complete E1 additions, the GK commitments from the commit kernel (E2); every s2 slot
    // is TOM_E2_WORDS wide, a derived point's (X, Y, Z) fills the first TOM_PROJ_WORDS of one
    launch_tom_norm(st, c.s2_proj + nj * TOM_E2_WORDS, nullptr, c.s2_bytes + nj * BSTRIDE, nd, 0, 1, 1, TOM_E2_WORDS);
  }
  if (gk) launch_tom_norm(st, c.s2_proj + g0 * TOM_E2_WORDS, nullptr, c.s2_bytes + g0 * BSTRIDE, ng, 1);
  if (items) {
    launch(st, M * HASHES_PER_ITEM, ItemHashTask{c});
    launch(st, M * 7, ItemEmitTask{c});
  }
}
// the verifier's Groth-Kohlweiss chain (gk.ts:197-262): ring polynomial, relations, offsets of the GK entries of the rows
void verify_gk(Stream& st, const VerifyCtx& c, uint32_t* gk_offs) {
  const int nblk = gk_blocks(c.n), ngk = 4 * c.n + 1;
  if (nblk > 1) launch(st, (long long)c.B * nblk, VGkSumTask{c});
  launch(st, c.B, VGkTask{c});
  launch(st, (long long)c.B * ngk, VGkOffsetsTask{c, gk_offs});
}

// The stage chain of one verifier chunk on lane `ln`, from VLayoutTask to VFinalTask, with the chunk-wide aggregate check
// first when `agg`.  c holds the chunk's inputs, ring and ok / status rows; its workspace is the lane's pool w (and the agg
// pools).  Every stage ends on the lane's stream.  b0: the chunk's first row in the call (hashed into the aggregate's
// weights); agg_c (may be null) receives the window bits of the tomEdwards256 aggregate MSM.  Returns the aggregate's
// control words on the device (null without it).
const uint32_t* verify_chunk(zka_ctx* ctx, Lane& ln, VerifyCtx& c, uint32_t b0, bool agg, int* agg_c) {
  Stream& st = ln.st;
  const int Bc = c.B, S = c.S, K = c.K, n = c.n, mode = c.mode;
  const size_t ns = (size_t)Bc * K;
  const int ET = c.ent_tom(), EN = c.ent_nist(), SG = c.segs();
  const int ngk = 4 * n + 1;
  Cursor w(ln.w);
  c.rep_off = w.take<uint32_t>((size_t)Bc * S);
  c.gk_off = w.take<uint32_t>(Bc);
  c.tagbits = w.take<uint32_t>((size_t)Bc * 3);
  c.chal = w.take<uint32_t>((size_t)Bc * 3);
  c.gk_ok_len = w.take<uint8_t>(Bc);
  c.r_aff = w.take<uint32_t>((size_t)Bc * 16);
  c.q_aff = w.take<uint32_t>((size_t)Bc * 16);
  c.q_inf = w.take<uint8_t>(Bc);
  c.rpows = w.take<uint32_t>((size_t)Bc * RT_NWIN * P256_PROJ_WORDS);
  c.rrows = w.take<uint32_t>((size_t)Bc * RT_ENTRIES * P256_PROJ_WORDS);
  c.rtab = w.take<uint32_t>((size_t)Bc * RT_ENTRIES * P256_AFF_WORDS);
  c.samp_idx = w.take<uint32_t>(ns);
  c.samp_draw = w.take<uint32_t>(ns);
  c.sp_T = w.take<uint32_t>(ns * P256_PROJ_WORDS);
  c.sp_T_aff = w.take<uint32_t>(ns * 16);
  c.sp_T_inf = w.take<uint8_t>(ns);
  c.ta_jv = w.take<uint32_t>(ns * 2 * 8);
  c.ta_jr = w.take<uint32_t>(ns * 2 * 8);
  c.ta_proj = w.take<uint32_t>(ns * 2 * TOM_E2_WORDS);
  c.ta_aff = w.take<uint32_t>(ns * 2 * TOM_AFF_WORDS);
  c.td_proj = w.take<uint32_t>(ns * DERS_PER_ITEM * TOM_PROJ_WORDS);
  c.td_aff = w.take<uint32_t>(ns * DERS_PER_ITEM * TOM_AFF_WORDS);
  c.td_bytes = w.take<uint8_t>(ns * DERS_PER_ITEM * BSTRIDE);
  c.item_chal = w.take<uint32_t>(ns * HASHES_PER_ITEM * 3);
  c.ent_scalar = w.take<uint32_t>((size_t)Bc * ET * 8);
  c.ent_off = w.take<uint32_t>((size_t)Bc * ET);
  c.ent_pre = w.take<uint32_t>((size_t)Bc * ET * TOM_PRE_WORDS);
  c.ent_cnt = w.take<uint32_t>(ns);
  c.part = w.take<uint32_t>(ns * V_PART_WORDS);
  // the small per-proof arrays before the entries and windows: the prover of this lane has small arrays at the
  // same places of the pool, so these share its buffers without growing them much
  c.fx_jv = w.take<uint32_t>((size_t)Bc * 2 * 8);
  c.fx_jr = w.take<uint32_t>((size_t)Bc * 2 * 8);
  c.fx_proj = w.take<uint32_t>((size_t)Bc * 2 * TOM_PROJ_WORDS);
  c.nfix = w.take<uint32_t>((size_t)Bc * P256_PROJ_WORDS);
  c.id_flags = w.take<uint8_t>((size_t)Bc * 3);
  c.gk_tape_bad = w.take_if<uint8_t>(mode == 0, Bc);
  c.vkey = w.take<int32_t>(Bc);
  c.nent_scalar = w.take<uint32_t>((size_t)Bc * EN * 8);
  c.nent_aff = w.take<uint32_t>((size_t)Bc * EN * 16);
  c.nent_skip = w.take<uint8_t>((size_t)Bc * EN);
  c.gk_scalar = w.take<uint32_t>((size_t)Bc * ngk * 8);
  c.gk_pre = w.take<uint32_t>((size_t)Bc * ngk * TOM_PRE_WORDS);
  uint32_t* gk_offs = w.take<uint32_t>((size_t)Bc * ngk);
  c.win_w = w.take<uint32_t>((size_t)Bc * SG * MSM_NWIN * 36);
  c.win_g = w.take<uint32_t>((size_t)Bc * MSM_NWIN * 36);
  c.win_n = w.take<uint32_t>((size_t)Bc * MSM_NWIN_N * P256_PROJ_WORDS);
  c.gk_part = w.take_if<uint32_t>(gk_blocks(n) > 1, (size_t)Bc * gk_blocks(n) * 8);
  const size_t agg_tape_len = verify_tape_len(n, S, K);
  const int agg_tp = agg_tape_pieces(agg_tape_len), agg_np = agg_tp + K + 1;
  uint32_t* agg_wt = w.take_if<uint32_t>(agg, (size_t)Bc * AGG_WT * 8);
  uint32_t* agg_dig = w.take_if<uint32_t>(agg, (size_t)Bc * agg_np * 8);
  c.chal_full = w.take_if<uint32_t>(agg, (size_t)Bc * 8);
  c.nfix_k = w.take_if<uint32_t>(agg, (size_t)Bc * 16);

  launch(st, Bc, VLayoutTask{c});
  launch(st, (long long)Bc * (S + 1), VValidateTask{c});
  {
    // the per-proof tables of R (a 255-doubling chain per proof, rows, normalisation: no status writes) run beside the
    // Fiat-Shamir hash of the repetitions (one thread per proof, 16 KB) unless per-kernel profiling is on
    const bool fork = !st.profiling;
    Stream& sr = fork ? ln.aux[0] : st;
    if (fork) { ev_record(ln.ev_fork, st); ev_wait(sr, ln.ev_fork); }
    launch(sr, Bc, P256PowsTask{c.r_aff, nullptr, c.rpows, Bc, RT_NWIN, RT_W});
    launch(sr, (long long)Bc * RT_NWIN, P256RowsSignedTask{c.rpows, c.rrows});
    launch_p256_norm(sr, c.rrows, c.rtab, nullptr, nullptr, (long long)Bc * RT_ENTRIES);
    launch(st, Bc, VChallengeTask{c});
    if (fork) { ev_record(ln.ev_join[0], sr); ev_wait(st, ln.ev_join[0]); }
  }
  // the Groth-Kohlweiss chain (ring polynomial, relations, offsets) only needs the layout: it runs on a side stream
  // beside the sampled-repetition chain; its tape-range status is folded in by VReduceTask (same precedence)
  const bool gk_fork = mode == 0 && !st.profiling;
  if (gk_fork) {
    ev_record(ln.ev_fork, st);
    ev_wait(ln.aux[1], ln.ev_fork);
  }
  if (agg) {
    // the aggregate's weights (zk_verify_agg.cuh) need the layout, the sampled repetitions and the exp challenge: they
    // hash ahead of the GK chain on its side stream (joined before VReduceTask)
    Stream& sw = gk_fork ? ln.aux[1] : st;
    launch(sw, (long long)Bc * agg_np, AggPieceTask{c, agg_tape_len, agg_tp, agg_np, agg_dig});
    launch(sw, Bc, AggWeightTask{c, c.chal_full, agg_dig, b0, agg_np, agg_wt});
  }
  if (gk_fork) {
    verify_gk(ln.aux[1], c, gk_offs);
    ev_record(ln.ev_join[1], ln.aux[1]);
  }
  launch(st, (long long)ns, VSampleP256Task{c});
  launch_p256_norm(st, c.sp_T, c.sp_T_aff, nullptr, c.sp_T_inf, (long long)(ns));
  launch(st, (long long)ns, VSampleJobsTask{c});
  launch(st, (long long)ns * 2, TomCommitTask{c.ta_jv, c.ta_jr, c.tg_tab, c.th_tab, c.ta_proj, c.tom});
  launch_tom_norm(st, c.ta_proj, c.ta_aff, nullptr, (long long)(ns * 2), 1);
  launch(st, (long long)ns, VDerivedTask{c});
  launch_tom_norm(st, c.td_proj, nullptr, c.td_bytes, (long long)(ns * DERS_PER_ITEM), 0);
  launch(st, (long long)ns * HASHES_PER_ITEM, VItemHashTask{c});
  dev_memset(st, c.ent_off, 0, (size_t)Bc * ET * 4);
  launch(st, (long long)ns, VRelationsTask{c});
  if (mode == 0) {
    if (gk_fork) ev_wait(st, ln.ev_join[1]);
    else verify_gk(st, c, gk_offs);
  }
  launch(st, Bc, VReduceTask{c});
  launch(st, (long long)Bc * ET, VParseEntriesTask{c.proofs, c.proof_stride, c.ent_off, c.ent_pre, ET});
  if (mode == 0) launch(st, (long long)Bc * ngk, VParseEntriesTask{c.proofs, c.proof_stride, gk_offs, c.gk_pre, ngk});
  launch(st, (long long)Bc * 2, TomCommitTask{c.fx_jv, c.fx_jr, c.tg_tab, c.th_tab, c.fx_proj, c.tom, 1});
  // chunk-wide aggregate check (zk_verify_agg.cuh): the sum over all proofs of the chunk of the three linear
  // combinations, as ONE wide-window MSM per group; when both sums are the identity the per-proof MSMs below
  // return at once
  uint32_t* ctl = nullptr;
  if (agg) {
    Cursor A(ln.agg);
    const int fgroups = (Bc * 2 + 63) / 64, ngroups = (Bc + 31) / 32, ngroups2 = (ngroups + 31) / 32;
    ctl = A.take<uint32_t>(AGG_CTL_WORDS);
#if !defined(ZKA_PG_WAR256)
    uint32_t* tpart = A.take<uint32_t>((size_t)Bc * (K + 2) * 2 * PG_EXT_WORDS);
#endif
    uint32_t* fpart = A.take<uint32_t>((size_t)fgroups * 16);
    uint32_t* fjv = A.take<uint32_t>(8);
    uint32_t* fjr = A.take<uint32_t>(8);
    uint32_t* fproj = A.take<uint32_t>(TOM_PROJ_WORDS);
    uint32_t* nfix_w = A.take<uint32_t>((size_t)Bc * P256_PROJ_WORDS);
    uint32_t* npart = A.take<uint32_t>((size_t)ngroups * P256_PROJ_WORDS);
    uint32_t* npart2 = A.take_if<uint32_t>(ngroups > 32, (size_t)ngroups2 * P256_PROJ_WORDS);
    dev_memset(st, ctl, 0, AGG_CTL_WORDS * 4);
    launch(st, Bc, AggGateTask{c, ctl});
    const AggTomSrc tsrc{c.ent_scalar, c.ent_pre, c.ent_cnt, c.gk_scalar, c.gk_pre, Bc, ET, K, ngk, agg_wt};
    const AggNistSrc nsrc{c.nent_scalar, c.nent_aff, c.nent_skip, Bc, EN, agg_wt};
    // three independent chains from here to AggFinalTask: the tomEdwards256 MSM (this stream), the torsion guard and the
    // P-256 MSM with its fixed parts (two side streams; with per-kernel profiling on, everything stays on one stream
    // so that the event pairs time one kernel at a time).  A skip flag raised by the torsion guard may reach the MSM
    // kernels late — they then only do work AggFinalTask discards.
    const bool fork = !st.profiling;
    Stream& sa = fork ? ln.aux[0] : st;
    Stream& sb = fork ? ln.aux[1] : st;
    if (fork) {
      ev_record(ln.ev_fork, st);
      ev_wait(sa, ln.ev_fork);
      ev_wait(sb, ln.ev_fork);
    }
#if !defined(ZKA_PG_WAR256)
    // cofactor 4: no small-order components, or the per-proof path decides
    launch(sa, (long long)Bc * (K + 2) * 2, AggTorsionPartTask{tsrc, ctl, tpart});
    launch(sa, (long long)Bc * 2, AggTorsionTask{tpart, ctl, K});
#endif
    const AggPlan tp = agg_plan((double)Bc * (0.5 * K * V_ENT_PER_SAMPLE + 2 + ngk), ctx->agg_c);
    const AggPlan np = agg_plan((double)Bc * EN, 0);
    if (agg_c) *agg_c = tp.D.c;
    const uint32_t *tA, *tB, *nA, *nB;
    agg_msm(st, Cursor(ln.agg_tom), tsrc, tp, ctl, &tA, &tB);
    agg_msm(sb, Cursor(ln.agg_nist), nsrc, np, ctl, &nA, &nB);
    // fixed-base parts: one commitment for the summed weighted tomEdwards256 scalars, a two-level sum of the weighted
    // P-256 points
    launch(st, fgroups, AggFixPartTask{ctl, c.fx_jv, c.fx_jr, agg_wt, fpart, Bc});
    launch(st, 1, AggFixSumTask{ctl, fpart, fjv, fjr, fgroups});
    launch(st, 1, TomCommitTask{fjv, fjr, c.tg_tab, c.th_tab, fproj, c.tom, 1});
    launch(sb, Bc, AggNistFixWeightTask{ctl, c.nfix_k, agg_wt, c.rtab, c.h_tab8, c.h_w, nfix_w});
    launch(sb, ngroups, AggNistFixPartTask{ctl, nfix_w, npart, Bc});
    int nleft = ngroups;            // second level: at most Bc / 1024 partial sums reach the final thread
    const uint32_t* nsum = npart;
    if (nleft > 32) {
      launch(sb, ngroups2, AggNistFixPartTask{ctl, npart, npart2, nleft});
      nsum = npart2;
      nleft = ngroups2;
    }
    if (fork) {
      ev_record(ln.ev_join[0], sa);
      ev_record(ln.ev_join[1], sb);
      ev_wait(st, ln.ev_join[0]);
      ev_wait(st, ln.ev_join[1]);
    }
    launch(st, 33, AggFinalTask{ctl, tA, tB, fproj, tp.D.nwin, tp.D.c, nA, nB, nsum, np.D.nwin, np.D.c, nleft});
    c.agg_ctl = ctl;
  }
  {
    const int nW = Bc * SG * MSM_NWIN, nWp = (nW + 31) & ~31, nG = Bc * MSM_NWIN;
    launch(st, (long long)nWp + nG,
           MsmTomWindowBothTask{MsmTomWindowTask{c.ent_scalar, c.ent_pre, c.ent_cnt, ET, K, V_ENT_PER_SAMPLE, 2, V_SEG, SG, c.win_w},
                                MsmTomWindowTask{c.gk_scalar, c.gk_pre, nullptr, ngk, 0, 0, mode == 0 ? ngk : 0, V_SEG, 1, c.win_g}, nW, nWp, nG, ctl});
  }
  launch(st, (long long)Bc * MSM_NWIN_N, MsmP256WindowTask{c.nent_scalar, c.nent_aff, c.nent_skip, c.win_n, EN, ctl});
  {
    const int Bp = (Bc + 31) & ~31;
    launch(st, 3ll * Bp, MsmCombineAllTask{MsmTomCombineTask{c.win_g, c.fx_proj, c.id_flags, 2, 0, 0},
                                           MsmTomCombineTask{c.win_w, c.fx_proj, c.id_flags, 2, 1, 1, SG},
                                           MsmP256CombineTask{c.win_n, c.nfix, c.id_flags}, Bc, Bp, ctl});
  }
  launch(st, Bc, VFinalTask{c});
  return ctl;
}

// The prover's self-check of one chunk (include/zkattest.h, "Self-checked proving"), on the lane's stream behind
// FinalizeTask: verifySignatureList with samples = sec_level over the rows pc just wrote, still on the device, against each
// row's own ring; rows the prover accepted and the check does not are released like a row the prover rejected
// (CheckReleaseTask).  key: k_b of row b at key + b * key_stride, key_len bytes; in: the chunk's inputs on the device;
// counts: the lane's [checked, failed] rows of the call.
void check_chunk(zka_ctx* ctx, const zka_params* P, Lane& ln, const ProveCtx& pc, const ProveRows& in, const RingSrc& ring,
                 const uint32_t* ring_m, const uint8_t* key, size_t key_stride, int key_len, uint32_t b0, uint32_t* counts) {
  Stream& st = ln.st;
  const int Bc = pc.B, S = pc.S, n = pc.n;
  const size_t tape_stride = verify_tape_len(n, S, S);   // a multiple of 16
  Cursor k(ln.chk);
  uint8_t* seeds = k.take<uint8_t>((size_t)Bc * 32);
  uint8_t* todo = k.take<uint8_t>(Bc);
  uint8_t* tape = k.take<uint8_t>((size_t)Bc * tape_stride);
  uint8_t* ok = k.take<uint8_t>(Bc);
  int32_t* vstatus = k.take<int32_t>(Bc);
  // c_b before the verifier's chain takes the pool w: a hedged call's seeds live there
  launch(st, Bc, CheckSeedTask{key, key_stride, key_len, pc.status, seeds, todo});
  VerifyCtx c = verify_ctx(ctx, P, Bc, S, pc.N, n, S, 0);
  c.msg_hash = in.msg_hash;
  c.proofs = pc.proofs;
  c.proof_stride = pc.proof_stride;
  c.proof_len = pc.proof_len;
  c.tape = tape;
  c.tape_stride = tape_stride;
  ring.fill(c, ring_m, in.ring_of);
  const SeedVerifyTapeTask vt{seeds, tape, tape_stride, n, S, S, c.ring_of, c.ring_depth};
  launch(st, (long long)Bc * vt.slots(), vt);
  c.ok = ok;
  c.status = vstatus;
  verify_chunk(ctx, ln, c, b0, ctx->agg != 0, nullptr);
  launch(st, (long long)Bc * FIN_PARTS, CheckReleaseTask{todo, ok, vstatus, pc.proofs, pc.proof_stride, pc.proof_len, pc.status, counts});
}

}  // namespace

// =============================================================================== C ABI
extern "C" {

int zka_version(void) { return 1; }

const char* zka_last_error(const zka_ctx* ctx) { return ctx ? ctx->err.c_str() : "null context"; }

uint64_t zka_launch_count(const zka_ctx* ctx) {
  if (!ctx) return 0;
  uint64_t n = ctx->st.launches + ctx->aux[0].launches + ctx->aux[1].launches;
  for (const auto& l : ctx->extra) n += l->st.launches + l->aux[0].launches + l->aux[1].launches;
  return n;
}

void* zka_get_stream(zka_ctx* ctx) {
#if !defined(ZKA_HOSTSIM)
  return ctx ? (void*)ctx->st.s : nullptr;
#else
  return nullptr;
#endif
}
int zka_set_profiling(zka_ctx* ctx, int enable) {
  if (!ctx) return ZKA_E_ARG;
  try {
    for (int i = 0; i < 1 + (int)ctx->extra.size(); i++) { sync(ctx->lane(i).st); ctx->lane(i).st.profiling = enable != 0; }
  } catch (...) { return ZKA_E_CUDA; }
  return 0;
}
int zka_profile_reset(zka_ctx* ctx) {
  if (!ctx) return ZKA_E_ARG;
  try {
    for (int i = 0; i < 1 + (int)ctx->extra.size(); i++) { sync(ctx->lane(i).st); ctx->lane(i).st.prof.clear(); }
  } catch (...) { return ZKA_E_CUDA; }
  return 0;
}
// knobs that may change between calls (tests, sweeps): "lanes", "chunk", "host_chunk", "agg", "agg_c", "self_check"
int zka_set_option(zka_ctx* ctx, const char* key, long value) {
  if (!ctx || !key || value < 1) return ZKA_E_ARG;
  const std::string k(key);
  return guarded(ctx, [&]() -> int {
    if (k == "lanes") {
      if (value > 8) return ZKA_E_ARG;
      while ((int)ctx->extra.size() + 1 < value) {
        auto l = std::make_unique<Lane>();
        stream_create(l->st);
        stream_create(l->cs_in);
        stream_create(l->cs_out);
        stream_create(l->aux[0]);
        stream_create(l->aux[1]);
        l->st.profiling = ctx->st.profiling;
        ctx->extra.push_back(std::move(l));
      }
      ctx->nlanes = (int)value;
    } else if (k == "chunk") {
      ctx->chunk = (int)value;
    } else if (k == "host_chunk") {
      ctx->host_chunk = (int)value;
    } else if (k == "agg") {          // 1: off, 2: on (values start at 1)
      ctx->agg = (int)value - 1;
    } else if (k == "self_check") {   // 1: off, 2: on
      if (value > 2) return ZKA_E_ARG;
      ctx->self_check = (int)value - 1;
    } else if (k == "agg_c") {
      if (value < 4 || value > 16) return ZKA_E_ARG;
      ctx->agg_c = (int)value;
    } else {
      return ZKA_E_ARG;
    }
    return 0;
  });
}
long long zka_stat(zka_ctx* ctx, const char* key) {
  if (!ctx || !key) return -1;
  const std::string k(key);
  std::lock_guard<std::mutex> g(ctx->stat_mu);
  if (k == "agg_pass") return (long long)ctx->agg_pass;
  if (k == "agg_fail") return (long long)ctx->agg_fail;
  if (k == "self_check_rows") return (long long)ctx->self_check_rows;
  if (k == "self_check_fail") return (long long)ctx->self_check_fail;
  if (k == "agg_c") return (long long)ctx->agg_c_last;        // window bits of the last tomEdwards256 aggregate MSM
  if (k == "tom_n_lo") return (long long)ctx->tom.n_lo;
  if (k == "tom_fallback") return ctx->tom_fallback ? 1 : 0;
  return -1;
}
size_t zka_profile_json(zka_ctx* ctx, char* buf, size_t cap) {
  if (!ctx) return 0;
  std::map<std::string, ProfEntry> all;
  try {
    for (int i = 0; i < 1 + (int)ctx->extra.size(); i++) {
      sync(ctx->lane(i).st);
      for (auto& kv : ctx->lane(i).st.prof) {
        ProfEntry& e = all[kv.first];
        e.launches += kv.second.launches; e.ms += kv.second.ms; e.items += kv.second.items;
      }
    }
  } catch (...) { return 0; }
  std::string j = "{";
  bool first = true;
  for (auto& kv : all) {
    char tmp[512];
    snprintf(tmp, sizeof tmp, "%s\"%s\": {\"launches\": %llu, \"ms\": %.6f, \"items\": %llu}", first ? "" : ", ",
             kv.first.c_str(), (unsigned long long)kv.second.launches, kv.second.ms,
             (unsigned long long)kv.second.items);
    j += tmp;
    first = false;
  }
  j += "}";
  if (buf && cap) {
    size_t n = std::min(cap - 1, j.size());
    memcpy(buf, j.data(), n);
    buf[n] = 0;
  }
  return j.size() + 1;
}
#if defined(ZKA_PG_WAR256)
static const char* const PROOF_GROUP = "war256";
#else
static const char* const PROOF_GROUP = "tomEdwards256";
#endif
int zka_proof_group(char* name, size_t cap, int* point_bytes, int* scalar_bytes) {
  const char* n = PROOF_GROUP;
  if (name && cap) {
    strncpy(name, n, cap - 1);
    name[cap - 1] = 0;
  }
  if (point_bytes) *point_bytes = WP;
  if (scalar_bytes) *scalar_bytes = WS;
  return 0;
}
int zka_set_progress(zka_ctx* ctx, volatile uint32_t* flags, uint32_t cap) {
  if (!ctx) return ZKA_E_ARG;
  ctx->progress = flags;
  ctx->progress_cap = flags ? cap : 0;
  return 0;
}
int zka_chunk_schedule(zka_ctx* ctx, uint32_t B, int host_buffers, uint32_t* off, uint32_t cap) {
  if (!ctx || !off || cap == 0) return ZKA_E_ARG;
  const std::vector<uint32_t> v = chunk_schedule(B, (uint32_t)(host_buffers ? std::min(ctx->chunk, ctx->host_chunk) : ctx->chunk), ctx->nlanes,
                                                 host_buffers != 0);
  if (v.size() > cap) return ZKA_E_ARG;
  for (size_t i = 0; i < v.size(); i++) off[i] = v[i];
  return (int)v.size() - 1;
}
int zka_lanes(const zka_ctx* ctx) { return ctx ? ctx->nlanes : 0; }
int zka_config(const zka_ctx* ctx, int* tom_w, int* tom_nwin, int* chunk) {
  if (!ctx) return ZKA_E_ARG;
  if (tom_w) *tom_w = ctx->tom.w;
  if (tom_nwin) *tom_nwin = ctx->tom.nwin;
  if (chunk) *chunk = ctx->chunk;
  return 0;
}

int zka_init(int device, zka_ctx** out) {
  if (!out) return ZKA_E_ARG;
  *out = nullptr;
#if !defined(ZKA_HOSTSIM)
  int ndev = 0;
  cudaError_t e = cudaGetDeviceCount(&ndev);
  if (e != cudaSuccess || ndev == 0 || device >= ndev) {
    cudaGetLastError();
    return ZKA_E_CUDA;   // no GPU: fail loudly, there is no CPU fallback
  }
#endif
  std::unique_ptr<zka_ctx> ctx(new zka_ctx());
  const int rc = guarded(ctx.get(), [&] {
#if !defined(ZKA_HOSTSIM)
    ZK_CUDA_CHECK(cudaSetDevice(device));
    ZK_CUDA_CHECK(cudaStreamCreateWithFlags(&ctx->st.s, cudaStreamNonBlocking));
#endif
    ctx->device = device;
    // shape of the proof-group tables: ZKA_TOM_W pins one width for all windows; otherwise ZKA_TOM_NWIN lookups
    [[maybe_unused]] bool tom_pinned = false;
    if (const char* e = getenv("ZKA_TOM_W")) {
      int w = atoi(e);
      if (w >= 2 && w <= 24) { ctx->tom = fb_uniform(w); tom_pinned = true; }
    }
#if !defined(ZKA_PG_WAR256)
    if (const char* e = tom_pinned ? nullptr : getenv("ZKA_TOM_NWIN")) {
      int n = atoi(e);
      if (n >= 11 && n <= 128) ctx->tom = fb_lookups(n);
    }
#endif
    if (const char* e = getenv("ZKA_TOM_TABLE_MAX")) ctx->tom_table_max = (size_t)strtoull(e, nullptr, 10);
    if (const char* e = getenv("ZKA_CHUNK")) {
      int c = atoi(e);
      if (c >= 1) ctx->chunk = c;
    }
    if (const char* e = getenv("ZKA_NORM_MODEL")) g_norm_model = atoi(e) != 0;
#if !defined(ZKA_HOSTSIM)
    {
      int sms = 0;
      if (cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device) == cudaSuccess && sms > 0) g_norm_slots = sms * 4;
    }
#endif
    if (const char* e = getenv("ZKA_HOST_CHUNK")) {
      int c = atoi(e);
      if (c >= 1) ctx->host_chunk = c;
    }
    stream_create(ctx->cs_in);
    stream_create(ctx->cs_out);
    stream_create(ctx->aux[0]);
    stream_create(ctx->aux[1]);
    {
      int lanes = 3;
#if defined(ZKA_HOSTSIM)
      lanes = 1;
#endif
      if (const char* e = getenv("ZKA_LANES")) lanes = atoi(e);
      if (lanes < 1) lanes = 1;
      if (lanes > 8) lanes = 8;
      if (zka_set_option(ctx.get(), "lanes", lanes) != 0) throw std::runtime_error("lanes");
    }
    if (const char* e = getenv("ZKA_TAPE_SPLIT")) ctx->tape_split = atoi(e) != 0;
    if (const char* e = getenv("ZKA_AGG")) ctx->agg = atoi(e);
    if (const char* e = getenv("ZKA_AGG_C")) {
      int c = atoi(e);
      if (c >= 4 && c <= 16) ctx->agg_c = c;
    }
    if (const char* e = getenv("ZKA_P256_HW")) {   // window bits of the P-256 G / NistGroup.h tables: 8..24
      int w = atoi(e);
      if (w >= 8 && w <= 24) ctx->p256_hw = w;
    }
    DevBuf gen;
    uint32_t* d_gen = gen.get<uint32_t>(16 + TOM_AFF_WORDS);
    launch(ctx->st, 1, GenAffTask{d_gen, d_gen + 16});
    build_p256_tab(ctx.get(), d_gen, ctx->g8, 8);
    build_p256_tab(ctx.get(), d_gen, ctx->gw, ctx->p256_hw);
#if defined(ZKA_PG_WAR256)
    build_tom_tab(ctx.get(), d_gen + 16, ctx->tg);
#else
    // g and every h table share one shape, so it is settled here: a shape given by its lookups is kept when the g table
    // and one table more (the first parameter set's h) can be allocated; otherwise (other work may hold the card's
    // memory) what was taken is freed and the context walks one lookup more, 12 for the default: 2.3 GB per base.  A
    // width pinned with ZKA_TOM_W is not replaced: it fails.
    try {
      DevBuf room;
      alloc_tom_tab(ctx.get(), room);
      build_tom_tab(ctx.get(), d_gen + 16, ctx->tg);
    } catch (const std::exception&) {
      if (tom_pinned || ctx->tom.nwin >= 128) throw;
#if !defined(ZKA_HOSTSIM)
      cudaGetLastError();   // the failed allocation is handled here
#endif
      ctx->tg.buf.release();
      ctx->tom = fb_lookups(ctx->tom.nwin + 1);
      ctx->tom_fallback = true;
      build_tom_tab(ctx.get(), d_gen + 16, ctx->tg);
    }
#endif
    // encoding of g (C_14 = params.g in pi_8, pointAdd.ts:144,220): normalise the table entry 1*g
    DevBuf proj, aff;
    uint32_t* d_proj = proj.get<uint32_t>(TOM_PROJ_WORDS);
    uint32_t* d_aff = aff.get<uint32_t>(TOM_AFF_WORDS);
    uint8_t* d_bytes = ctx->tg_bytes.get<uint8_t>(BSTRIDE);
    launch(ctx->st, 1, GProjTask{d_gen + 16, d_proj});
    launch_tom_norm(ctx->st, d_proj, d_aff, d_bytes, 1, 0);
    sync(ctx->st);
    return 0;
  });
  if (rc) {
    fprintf(stderr, "zka_init: %s\n", ctx->err.c_str());
    return rc;
  }
  *out = ctx.release();
  return 0;
}

void zka_shutdown(zka_ctx* ctx) { delete ctx; }

int zka_params_create(zka_ctx* ctx, const uint8_t h_nist[65], const uint8_t h_proof[67], uint32_t sec_level,
                      zka_params** out) {
  if (!ctx || !h_nist || !h_proof || !out) return ZKA_E_ARG;
  if (sec_level < 1 || sec_level > MAX_REPS) return fail(ctx, ZKA_E_ARG, "sec_level must be in [1,80]");
  return guarded(ctx, [&] {
    std::unique_ptr<zka_params> P(new zka_params());
    P->ctx = ctx;
    P->sec_level = sec_level;
    P->h_w = ctx->p256_hw;
    memcpy(P->h_nist, h_nist, 65);
    memcpy(P->h_proof, h_proof, WP);
    {   // SHA-256("ZKAttest/hedge/params/v1" || group name NUL-padded to 16 || h_nist || h_proof || le32(sec_level))
      uint8_t name[16] = {};
      memcpy(name, PROOF_GROUP, strlen(PROOF_GROUP));
      Sha256 h;
      h.init();
      sha_tag(h, "ZKAttest/hedge/params/v1");
      h.update(name, 16);
      h.update(h_nist, 65);
      h.update(h_proof, WP);
      h.put4(sec_level);
      alignas(16) uint8_t d[32];
      sha_store(h, d);
      memcpy(P->hedge_digest, d, 32);
    }
    DevBuf bn, bt, an, at, bad, inf;
    uint8_t* d_bn = bn.get<uint8_t>(65);
    uint8_t* d_bt = bt.get<uint8_t>(WP);
    uint32_t* d_an = an.get<uint32_t>(16);
    uint32_t* d_at = at.get<uint32_t>(TOM_AFF_WORDS);
    uint8_t* d_bad = bad.get<uint8_t>(2);
    uint8_t* d_inf = inf.get<uint8_t>(1);
    copy_h2d(ctx->st, d_bn, h_nist, 65);
    copy_h2d(ctx->st, d_bt, h_proof, WP);
    launch(ctx->st, 1, ParsePointsTask{d_bn, nullptr, d_an, nullptr, d_bad, d_inf});
    launch(ctx->st, 1, ParsePointsTask{nullptr, d_bt, nullptr, d_at, d_bad + 1, nullptr});
    uint8_t hb[3];
    copy_d2h(ctx->st, hb, d_bad, 2);
    copy_d2h(ctx->st, hb + 2, d_inf, 1);
    sync(ctx->st);
    if (hb[0] || hb[1] || hb[2]) return fail(ctx, ZKA_E_ARG, "params: h point not on its group");
    build_p256_tab(ctx, d_an, P->h8, P->h_w);
    build_tom_tab(ctx, d_at, P->th);
    *out = P.release();
    return 0;
  });
}

void zka_params_destroy(zka_params* P) { delete P; }

// R rings in one device handle: the keys cross once, and one RingSetPrepTask launch prepares every ring of the set
int zka_rings_create(zka_ctx* ctx, uint32_t R, const uint32_t* sizes, const uint8_t* keys, zka_rings** out) {
  if (!ctx || !sizes || !keys || !out) return ZKA_E_ARG;
  *out = nullptr;
  if (R == 0) return fail(ctx, ZKA_E_ARG, "a ring set holds at least one ring");
  // every ring takes at least 2 padded entries
  if (R > (1u << 23)) return fail(ctx, ZKA_E_ARG, "ring set exceeds 2^24 padded entries");
  std::unique_ptr<zka_rings> set(new zka_rings());
  set->ctx = ctx;
  set->R = R;
  std::vector<uint32_t> key_off(R), base(R);
  uint64_t nkeys = 0, total = 0;
  for (uint32_t r = 0; r < R; r++) {
    const uint32_t N = sizes[r];
    if (N < 2 || N > (1u << 20)) return fail(ctx, ZKA_E_ARG, "ring size must be in [2, 2^20]");
    const int n = ceil_log2(N);
    set->size.push_back(N);
    set->depth.push_back(n);
    key_off[r] = (uint32_t)nkeys;
    base[r] = (uint32_t)total;
    nkeys += N;
    total += 1ull << n;
    if (total > (1ull << 24)) return fail(ctx, ZKA_E_ARG, "ring set exceeds 2^24 padded entries");
  }
  return guarded(ctx, [&] {
    Stream& st = ctx->st;
    DevBuf kbuf, obuf;
    const uint8_t* d_keys = stage_in(st, kbuf, keys, (size_t)nkeys * 32);
    uint32_t* d_off = obuf.get<uint32_t>(R);
    uint32_t* d_base = set->ring_base.get<uint32_t>(R);
    uint32_t* d_size = set->ring_size.get<uint32_t>(R);
    uint32_t* d_depth = set->ring_depth.get<uint32_t>(R);
    const std::vector<uint32_t> depth(set->depth.begin(), set->depth.end());
    const int nmax = *std::max_element(set->depth.begin(), set->depth.end());
    uint32_t* ring_m = set->ring_m.get<uint32_t>((size_t)total * 8);
    copy_h2d(st, d_off, key_off.data(), (size_t)R * 4);
    copy_h2d(st, d_base, base.data(), (size_t)R * 4);
    copy_h2d(st, d_size, set->size.data(), (size_t)R * 4);
    copy_h2d(st, d_depth, depth.data(), (size_t)R * 4);
    launch(st, (long long)total, RingSetPrepTask{d_keys, d_off, d_base, d_size, ring_m, (int)R});
    launch(st, nmax, GkLagrangeSetTask{set->lag.get<uint32_t>(ProveCtx::gk_lag_off(nmax + 1))});
    // the hedge digest of every ring (RingDigestTask), for the hedged prove calls
    std::vector<uint32_t> leaf_off(R + 1, 0);
    for (uint32_t r = 0; r < R; r++) leaf_off[r + 1] = leaf_off[r] + hedge_leaves(set->depth[r]);
    DevBuf lbuf, leaves;
    uint32_t* d_leaf_off = lbuf.get<uint32_t>(R + 1);
    copy_h2d(st, d_leaf_off, leaf_off.data(), (size_t)(R + 1) * 4);
    RingDigestTask dt{ring_m, d_base, d_size, d_depth, d_leaf_off, 0u, 0u, R, leaves.get<uint8_t>((size_t)32 * leaf_off[R]),
                      set->ring_digest.get<uint8_t>((size_t)32 * R), false};
    launch(st, leaf_off[R], dt);
    dt.root = true;
    launch(st, R, dt);
    sync(st);
    *out = set.release();
    return 0;
  });
}

void zka_rings_destroy(zka_rings* set) { delete set; }

size_t zka_proof_max_len(uint32_t ring_size, uint32_t sec_level) {
  return (size_t)proof_len((int)sec_level, ceil_log2(ring_size), (int)sec_level);
}
size_t zka_prove_tape_len(uint32_t ring_size, uint32_t sec_level) {
  return (size_t)32 * prove_draws((int)sec_level, ceil_log2(ring_size), (int)sec_level);
}
size_t zka_verify_tape_len(uint32_t ring_size, uint32_t sec_level) {
  return verify_tape_len(ceil_log2(ring_size), (int)sec_level);
}

// ------------------------------------------------------------------------------ sub-ops
int zka_tom_commit_batch(zka_ctx* ctx, const zka_params* P, uint32_t count, const uint8_t* v, const uint8_t* r,
                         uint8_t* out) {
  if (!ctx || !P || !v || !r || !out) return ZKA_E_ARG;
  if (count == 0) return 0;
  return guarded(ctx, [&] {
    Stream& st = ctx->st;
    Cursor in(ctx->in[0]), w(ctx->w), ob(ctx->out[0]);
    const uint8_t* dv = stage_in(st, in.next(), v, (size_t)count * 32);
    const uint8_t* dr = stage_in(st, in.next(), r, (size_t)count * 32);
    uint32_t* jv = w.take<uint32_t>((size_t)count * 8);
    uint32_t* jr = w.take<uint32_t>((size_t)count * 8);
    uint32_t* proj = w.take<uint32_t>((size_t)count * TOM_E2_WORDS);
    uint32_t* aff = w.take<uint32_t>((size_t)count * TOM_AFF_WORDS);
    uint8_t* bytes = w.take<uint8_t>((size_t)count * BSTRIDE);
    const Output<uint8_t> o(out, WP);
    uint8_t* packed = o.rows(ob.next(), 0, count);
    launch(st, count, CommitConvTask{dv, dr, jv, jr});
    launch(st, count, TomCommitTask{jv, jr, ctx->tg.tab, P->th.tab, proj, ctx->tom});
    launch_tom_norm(st, proj, aff, bytes, (long long)(count), 1);
    launch(st, count, PackTomTask{bytes, packed});
    o.copy_back(st, 0, packed, count);
    sync(st);
    return 0;
  });
}

int zka_p256_mul_batch(zka_ctx* ctx, uint32_t count, const uint8_t* base, const uint8_t* k, uint8_t* out) {
  if (!ctx || !k || !out) return ZKA_E_ARG;
  if (count == 0) return 0;
  return guarded(ctx, [&] {
    Stream& st = ctx->st;
    Cursor in(ctx->in[0]), w(ctx->w), ob(ctx->out[0]);
    const uint8_t* dk = stage_in(st, in.next(), k, (size_t)count * 32);
    const uint8_t* db = stage_in(st, in.next(), base, (size_t)count * 65);
    uint32_t* proj = w.take<uint32_t>((size_t)count * P256_PROJ_WORDS);
    uint32_t* aff = w.take<uint32_t>((size_t)count * P256_AFF_WORDS);
    uint8_t* bytes = w.take<uint8_t>((size_t)count * BSTRIDE);
    uint8_t* inf = w.take<uint8_t>(count);
    // with a base per row: per-base w=4 positional tables, the same path the prover uses for R (PhaseAP256Task)
    const bool per_base = db != nullptr;
    uint32_t* baff = w.take_if<uint32_t>(per_base, (size_t)count * 16);
    uint8_t* bad = w.take_if<uint8_t>(per_base, count);
    uint8_t* binf = w.take_if<uint8_t>(per_base, count);
    uint32_t* pows = w.take_if<uint32_t>(per_base, (size_t)count * RT_NWIN * P256_PROJ_WORDS);
    uint32_t* rows = w.take_if<uint32_t>(per_base, (size_t)count * RT_ENTRIES * P256_PROJ_WORDS);
    uint32_t* rtab = w.take_if<uint32_t>(per_base, (size_t)count * RT_ENTRIES * P256_AFF_WORDS);
    const Output<uint8_t> o(out, NP);
    uint8_t* packed = o.rows(ob.next(), 0, count);
    if (per_base) {
      launch(st, count, ParsePointsTask{db, nullptr, baff, nullptr, bad, binf});
      launch(st, count, P256PowsTask{baff, binf, pows, (int)count, RT_NWIN, RT_W});
      launch(st, (long long)count * RT_NWIN, P256RowsSignedTask{pows, rows});
      const long long np = (long long)count * RT_ENTRIES;
      launch_p256_norm(st, rows, rtab, nullptr, nullptr, (long long)(np));
    }
    launch(st, count, P256MulTask{dk, ctx->g8.tab, rtab, binf, proj});
    launch_p256_norm(st, proj, aff, bytes, inf, (long long)(count));
    launch(st, count, PackP256Task{bytes, packed});
    o.copy_back(st, 0, packed, count);
    sync(st);
    return 0;
  });
}


int zka_field_op_batch(zka_ctx* ctx, int field, int op, uint32_t count, const uint8_t* a, const uint8_t* b,
                       uint8_t* out) {
  if (!ctx || !a || !out || field < 0 || field > 2 || op < 0 || op > 4 || (op < 3 && !b)) return ZKA_E_ARG;
  if (count == 0) return 0;
  return guarded(ctx, [&] {
    Stream& st = ctx->st;
    Cursor in(ctx->in[0]), ob(ctx->out[0]);
    const int nb = field == 2 ? WCB : 32;
    const uint8_t* da = stage_in(st, in.next(), a, (size_t)count * nb);
    const uint8_t* db = stage_in(st, in.next(), b, (size_t)count * nb);
    const Output<uint8_t> o(out, nb);
    uint8_t* dout = o.rows(ob.next(), 0, count);
    if (field == 0) launch(st, count, FieldOpTask<P256p, 32>{da, db, dout, op});
    else if (field == 1) launch(st, count, FieldOpTask<P256n, 32>{da, db, dout, op});
    else launch(st, count, FieldOpTask<PGp, WCB>{da, db, dout, op});
    o.copy_back(st, 0, dout, count);
    sync(st);
    return 0;
  });
}

int zka_hash80_batch(zka_ctx* ctx, uint32_t count, const uint8_t* msgs, size_t msg_stride, const uint32_t* len,
                     uint8_t* out) {
  if (!ctx || !msgs || !len || !out) return ZKA_E_ARG;
  if (count == 0) return 0;
  return guarded(ctx, [&] {
    Stream& st = ctx->st;
    Cursor in(ctx->in[0]), ob(ctx->out[0]);
    const uint8_t* dm = stage_in(st, in.next(), msgs, (size_t)count * msg_stride);
    const uint32_t* dl = stage_in(st, in.next(), len, (size_t)count);
    const Output<uint8_t> o(out, 10);
    uint8_t* dout = o.rows(ob.next(), 0, count);
    launch(st, count, Hash80Task{dm, msg_stride, dl, dout});
    o.copy_back(st, 0, dout, count);
    sync(st);
    return 0;
  });
}

int zka_params_generate(zka_ctx* ctx, const uint8_t rnd[64], uint8_t h_nist[65], uint8_t h_proof[67]) {
  if (!ctx || !rnd || !h_nist || !h_proof) return ZKA_E_ARG;
  return guarded(ctx, [&] {
    // h_nist = G * rnd0 (pedersen.ts:66-67 on p256); h_proof = g * rnd1 + 0 * g
    int rc = zka_p256_mul_batch(ctx, 1, nullptr, rnd, h_nist);
    if (rc) return rc;
    Stream& st = ctx->st;
    Cursor in(ctx->in[0]), w(ctx->w);
    uint32_t* jv = w.take<uint32_t>(8);
    uint32_t* jr = w.take<uint32_t>(8);
    uint32_t* proj = w.take<uint32_t>(TOM_E2_WORDS);
    uint32_t* aff = w.take<uint32_t>(TOM_AFF_WORDS);
    uint8_t* bytes = w.take<uint8_t>(BSTRIDE);
    uint8_t* d_rnd = in.take<uint8_t>(32);
    copy_h2d(st, d_rnd, rnd + 32, 32);
    launch(st, 1, GenConvTask{d_rnd, jv, jr});
    // v*g + 0*g: use the g table for both bases
    launch(st, 1, TomCommitTask{jv, jr, ctx->tg.tab, ctx->tg.tab, proj, ctx->tom});
    launch_tom_norm(st, proj, aff, bytes, (long long)(1), 1);
    copy_d2h(st, h_proof, bytes, WP);
    sync(st);
    return 0;
  });
}

int zka_key_to_int(zka_ctx* ctx, uint32_t count, const uint8_t* pk, uint8_t* x_out, int32_t* status) {
  if (!ctx || !pk || !x_out) return ZKA_E_ARG;
  if (count == 0) return 0;
  return guarded(ctx, [&] {
    Stream& st = ctx->st;
    Cursor in(ctx->in[0]), w(ctx->w), ob(ctx->out[0]);
    const uint8_t* dp = stage_in(st, in.next(), pk, (size_t)count * 65);
    uint32_t* aff = w.take<uint32_t>((size_t)count * 16);
    uint8_t* bad = w.take<uint8_t>(count);
    uint8_t* inf = w.take<uint8_t>(count);
    const Output<uint8_t> xo(x_out, 32);
    const Output<int32_t> so(status, 1);   // status is optional: without it the statuses stay in the staging buffer
    uint8_t* dx = xo.rows(ob.next(), 0, count);
    int32_t* ds = so.rows(ob.next(), 0, count);
    launch(st, count, ParsePointsTask{dp, nullptr, aff, nullptr, bad, inf});
    launch(st, count, KeyToIntTask{aff, bad, inf, dx, ds});
    xo.copy_back(st, 0, dx, count);
    if (status) so.copy_back(st, 0, ds, count);
    sync(st);
    return 0;
  });
}

// ------------------------------------------------------------------------------- prove
// mode 0: proveSignatureList.  mode 1: proveExp alone (exp.ts:126-231) — base / s_in / q_in are the statement,
// msg_hash / sig / which are unused, the rows hold the repetitions only.
// seeds (B x 32, mode 0 only) instead of a tape: every lane expands its chunk's draws into its own tape buffer
// (SeedProveTapeTask), the draws before the challenge first, the item and GK draws after the scan.  hedge: the seeds
// SeedProveTapeTask reads are first derived per row (SeedHedgeTask) into a lane buffer; rows.seeds may then be null.
static int prove_impl(zka_ctx* ctx, const zka_params* P, uint32_t B, const ProveRows& rows, const RingSrc& ring, int mode) {
  const int S = (int)P->sec_level, n = ring.n;
  const bool hedge = rows.hedge, seeded = rows.seeds != nullptr || hedge;
  const bool check = ctx->self_check && mode == 0;
  // seeded: the library's tape rows hold every draw a proof can read (a multiple of 32 bytes, so 16-byte aligned rows)
  const int seed_draws = prove_draws(S, n, S);
  const uint32_t* ring_m = ring.prepare(ctx, true, hedge);
  const uint8_t* ring_digest = hedge ? ring.digests(ctx) : nullptr;
  const Output<uint8_t> po(rows.proofs, rows.proof_stride);
  const Output<uint32_t> lo(rows.proof_len, 1);
  const Output<int32_t> so(rows.status, 1);
  const int lanes = ctx->nlanes;
  const size_t dev_tape_stride = (rows.tape_stride + 15) & ~(size_t)15;   // row pitch of a host tape staged on the device
  // (hedged calls without caller seeds count as device memory: no randomness crosses PCIe)
  const uint8_t* rnd_in = seeded ? rows.seeds : rows.tape;
  const bool all_dev = po.dev && (!rnd_in || is_device_ptr(rnd_in));
  const std::vector<uint32_t> off = chunk_schedule(B, (uint32_t)(all_dev ? ctx->chunk : std::min(ctx->chunk, ctx->host_chunk)), lanes, !all_dev);
  const uint32_t nchunks = (uint32_t)off.size() - 1;
  const int used = (int)std::min<uint32_t>((uint32_t)lanes, nchunks);
  const bool trace = getenv("ZKA_TRACE") != nullptr;
  const auto t_call = std::chrono::steady_clock::now();
  auto ms_now = [&] { return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t_call).count(); };
  std::atomic<uint32_t> next_chunk((uint32_t)used);
  // Every lane claims chunks from a shared counter (one ahead of the one it is computing, so that its inputs are
  // already on their way).  Within a lane, chunks are software-pipelined over three streams when buffers live in
  // host memory (staging buffers double-buffered by slot).
  auto run_lane = [&](int li) {
    Lane& ln = ctx->lane(li);
    Stream& st = ln.st;
    ProveRows cin[2];   // each slot's chunk, its inputs on the device
    uint32_t* check_counts = check ? ln.chk_count.get<uint32_t>(2) : nullptr;   // copied back once, at the end of the call
    if (check) dev_memset(st, check_counts, 0, 8);
    auto issue_inputs = [&](uint32_t k, int slot) {
      // the chunk's rows of an input: from its first row to the next chunk's
      const ProveRows r = rows.at(off[k]), e = rows.at(off[k + 1]);
      const size_t Bc = off[k + 1] - off[k];
      Stream& ci = ln.cs_in;
      Cursor in(ln.in[slot]);
      DevBuf& tape_buf = in.next();   // first, like the verifier's proof rows: the largest inputs share one buffer
      auto stage = [&](auto* p, auto* end) { return stage_in(ci, in.next(), p, (size_t)(end - p)); };
      ev_wait(ci, ln.ev_done[slot]);   // the chunk that used these staging buffers before has finished reading them
      ProveRows& d = cin[slot];
      d.msg_hash = stage(r.msg_hash, e.msg_hash);
      d.sig = stage(r.sig, e.sig);
      d.pk = stage(r.pk, e.pk);
      d.which = stage(r.which, e.which);
      d.ring_of = stage(r.ring_of, e.ring_of);
      d.base = stage(r.base, e.base);
      d.s_in = stage(r.s_in, e.s_in);
      d.q_in = stage(r.q_in, e.q_in);
      d.seeds = stage(r.seeds, e.seeds);
      ev_record(ln.ev_small[slot], ci);
      if (seeded) {
        // filled on the lane's stream by SeedProveTapeTask; nothing crosses PCIe
        d.tape = tape_buf.get<uint8_t>(Bc * (size_t)32 * seed_draws);
      } else if (is_device_ptr(rows.tape)) {
        d.tape = r.tape;
      } else if (!ctx->tape_split && dev_tape_stride == rows.tape_stride) {
        d.tape = stage_in(ci, tape_buf, r.tape, (size_t)(e.tape - r.tape));
      } else {
        // host tape: staged at a row pitch of a multiple of 16 (dev_tape_stride), so that every draw is read with
        // 16-byte loads whatever the caller's stride.  With tape_split only the draws used before the challenge
        // (3 + 4S of up to 3 + 44S + 5n) travel now; the item and GK draws of each proof follow after the challenge,
        // when their number is known
        uint8_t* dt = tape_buf.get<uint8_t>(Bc * dev_tape_stride);
        const size_t width = ctx->tape_split ? std::min(rows.tape_stride, (size_t)32 * draws_before_items(S)) : rows.tape_stride;
        copy_d2h_2d(ci, dt, dev_tape_stride, r.tape, rows.tape_stride, width, Bc);
        d.tape = dt;
      }
      ev_record(ln.ev_tape[slot], ci);
    };
    // the first `used` chunks are dealt statically (lane threads start at slightly different times); later ones are
    // claimed from the shared counter at the mid-pipeline synchronisation point of the current chunk, when about
    // half of its kernels are queued: early enough for the next inputs to travel behind them, late enough that a
    // lane that started first does not grab the chunks of lanes that are still starting
    uint32_t k = (uint32_t)li;
    int slot = 0;
    if (k < nchunks) issue_inputs(k, slot);
    for (; k < nchunks; slot ^= 1) {
      const uint32_t b0 = off[k];
      const int Bc = (int)(off[k + 1] - b0);
      const uint32_t k_this = k;
      const double t_begin = ms_now();
      ev_wait(st, ln.ev_small[slot]);
      ev_wait(st, ln.ev_out[slot]);    // the proofs of chunk k-2 have left the output staging buffers
      ProveCtx c = prove_ctx(ctx, P, Bc, S, (int)ring.N, n);
      c.mode = mode; c.head_len = mode == 0 ? HEAD_LEN : 0;
      c.base = cin[slot].base; c.s_in = cin[slot].s_in; c.q_in = cin[slot].q_in;
      c.msg_hash = cin[slot].msg_hash;
      c.sig = cin[slot].sig;
      c.pk = cin[slot].pk;
      c.which = cin[slot].which;
      c.tape = cin[slot].tape;
      c.tape_stride = seeded ? (size_t)32 * seed_draws : is_device_ptr(rows.tape) ? rows.tape_stride : dev_tape_stride;
      c.tape_draws = seeded ? (uint32_t)seed_draws : (uint32_t)(rows.tape_stride / 32);
      ring.fill(c, ring_m, cin[slot].ring_of);
      const size_t S1 = (size_t)S + 1;
      const size_t nA = (size_t)Bc * S1;
      const size_t n1 = (size_t)Bc * (2 + 2 * S);
      Cursor w(ln.w);
      c.s1 = w.take<uint32_t>((size_t)Bc * 8);
      c.pk_aff = w.take<uint32_t>((size_t)Bc * 16);
      c.q_aff = w.take<uint32_t>((size_t)Bc * 16);
      c.q_inf = w.take<uint8_t>(Bc);
      c.r_aff = w.take<uint32_t>((size_t)Bc * 16);
      c.r_bytes = w.take<uint8_t>((size_t)Bc * BSTRIDE);
      c.rpows = w.take<uint32_t>((size_t)Bc * RT_NWIN * P256_PROJ_WORDS);
      c.rrows = w.take<uint32_t>((size_t)Bc * KEY_CAP * P256_PROJ_WORDS);
      c.rtab = w.take<uint32_t>((size_t)Bc * KEY_CAP * P256_AFF_WORDS);
      c.pa_T = w.take<uint32_t>(nA * P256_PROJ_WORDS);
      c.pa_A = w.take<uint32_t>(nA * P256_PROJ_WORDS);
      c.pa_T_aff = w.take<uint32_t>(nA * 16);
      c.pa_T_inf = w.take<uint8_t>(nA);
      c.pa_A_aff = w.take<uint32_t>(nA * 16);
      c.pa_A_bytes = w.take<uint8_t>(nA * BSTRIDE);
      c.pa_A_inf = w.take<uint8_t>(nA);
      c.s1_jv = w.take<uint32_t>(n1 * 8);
      c.s1_jr = w.take<uint32_t>(n1 * 8);
      c.s1_proj = w.take<uint32_t>(n1 * TOM_E2_WORDS);
      c.s1_aff = w.take<uint32_t>(n1 * TOM_AFF_WORDS);
      c.s1_bytes = w.take<uint8_t>(n1 * BSTRIDE);
      c.chal = w.take<uint32_t>((size_t)Bc * 3);
      c.zcount = w.take<uint32_t>(Bc);
      c.item_base = w.take<uint32_t>(Bc);
      c.item_total = w.take<uint32_t>(2);
      c.rep_off = w.take<uint32_t>((size_t)Bc * S);
      c.gk_off = w.take<uint32_t>(Bc);
      c.gk_dv = w.take<uint32_t>((size_t)Bc * n * 8);
      c.gk_x = w.take<uint32_t>((size_t)Bc * 3);
      c.u12 = w.take<uint32_t>((size_t)Bc * 16);
      c.tab_of = w.take<uint32_t>(Bc);
      c.tab_rep = w.take<uint32_t>((size_t)Bc * 2);
      c.tab_count = w.take<uint32_t>(2);
      c.which_s = w.take<uint32_t>(Bc);
      uint32_t* base_aff = w.take_if<uint32_t>(mode == 1, (size_t)Bc * 16);
      c.base_aff = mode == 0 ? c.pk_aff : base_aff;
      uint8_t* hedged = w.take_if<uint8_t>(hedge, (size_t)Bc * 32);
      const uint8_t* seeds = hedge ? hedged : cin[slot].seeds;   // what SeedProveTapeTask expands
      c.proof_stride = rows.proof_stride;
      Cursor ob(ln.out[slot]);
      c.proofs = po.rows(ob.next(), b0, Bc);
      c.proof_len = lo.rows(ob.next(), b0, Bc);
      c.status = so.rows(ob.next(), b0, Bc);

      // --- statement + per-proof tables of pk, then R = u1*G + u2*pk on the tables
      launch(st, Bc, PreKeyTask{c});
      // one table per DISTINCT key of the chunk (grids are sized for Bc tables, surplus threads return)
      launch(st, Bc, KeyDedupTask{c});
      launch(st, Bc, KeyRankTask{c});
      launch(st, Bc, KeyAssignTask{c});
      {
        const int Bp = (Bc + 31) & ~31;
        launch(st, (long long)Bp + Bc,
               PowsAndPreTask{P256PowsTask{c.base_aff, nullptr, c.rpows, Bc, RT_NWIN, RT_W, c.tab_rep, c.tab_count, c.tab_count + 1}, PreTask{c}, Bp});
      }
      // the window bits of these tables are chosen on the device from the number of distinct keys (tab_count[1]);
      // grids are sized for the worst case, surplus threads return
      // (one thread per (key, window, block of 16 entries): keys x windows x blocks <= Bc x KEY_CAP / 16 by the memory
      // rule of key_window_bits, e.g. 0.2 Bc keys x 33 x 8 at w = 8 or Bc x 52 x 1 at w = 5)
      launch(st, (long long)Bc * ((KEY_CAP + 15) / 16), P256RowsBlockTask{c.rpows, c.rrows, KEY_W_MIN, c.tab_count, c.tab_count + 1});
      {
        const long long np = (long long)Bc * KEY_CAP;
        // points per thread from the EXPECTED table volume (at most min(N, Bc) distinct keys when every key is a member
        // of the one ring; up to Bc with a ring set); the grid still covers the worst case
        const uint32_t kest = ring.set ? (uint32_t)Bc : std::min<uint32_t>(ring.N, (uint32_t)Bc);
        const int west = key_window_bits(kest, (uint32_t)Bc, (uint32_t)S + 2);
        const int ch = norm_chunk_for((long long)kest * fb_windows(west) * fb_entries(west), 5);
        launch(st, (np + ch - 1) / ch, P256NormTask{c.rrows, c.rtab, nullptr, nullptr, (int)np, ch, c.tab_count, 0, c.tab_count + 1});
      }
      // --- phase A (first consumer of the tape) and R = u1*G + u2*pk side by side
      ev_wait(st, ln.ev_tape[slot]);
      if (hedge) {
        SeedHedgeTask ht{{}, ring_digest, cin[slot].ring_of, cin[slot].seeds, c.msg_hash, c.sig, c.pk, c.which, hedged};
        memcpy(ht.params_digest, P->hedge_digest, 32);
        launch(st, Bc, ht);
      }
      if (seeded) {
        const int d1 = draws_before_items(S);
        launch(st, (long long)Bc * d1, SeedProveTapeTask{seeds, const_cast<uint8_t*>(c.tape), c.tape_stride, S, n, 0, d1, nullptr});
      }
      {
        const int nAp = (int)((nA + 31) & ~(size_t)31);
        launch(st, (long long)nAp + Bc, PhaseAAndRPointTask{PhaseAP256Task{c}, RPointTask{c}, (int)nA, nAp});
      }
      launch_p256_norm(st, c.pa_T, c.pa_T_aff, nullptr, c.pa_T_inf, (long long)(nA));
      launch_p256_norm(st, c.pa_A, c.pa_A_aff, c.pa_A_bytes, c.pa_A_inf, (long long)(nA));
      if (mode == 1) launch(st, Bc, ExpStatementTask{c});
      prove_store1(st, c);
      // --- challenge, layout
      launch(st, Bc, ExpChallengeTask{c});
      launch(st, 1, ScanTask{c});
      uint32_t tot2[2] = {0, 0};
      copy_d2h(st, tot2, c.item_total, 8);
      const bool tape_host = !seeded && ctx->tape_split && !is_device_ptr(rows.tape);
      sync(st);
      if (seeded) {
        // the item and GK draws of each proof, up to the longest a proof of the chunk can be (zmax = tot2[1], depth n)
        const int d1 = draws_before_items(S), span = prove_draws((int)tot2[1], n, S) - d1;
        launch(st, (long long)Bc * span,
               SeedProveTapeTask{seeds, const_cast<uint8_t*>(c.tape), c.tape_stride, S, n, d1, span, c.zcount, c.ring_of, c.ring_depth});
      } else if (tape_host) {
        // second part of the tape: draws [3 + 4S, 3 + 4S + 40 zmax + 5n) of every row in one strided copy
        // (zmax = the largest zero-bit count of the chunk)
        const size_t o0 = (size_t)32 * draws_before_items(S);
        const size_t o1 = std::min(rows.tape_stride, (size_t)32 * prove_draws((int)tot2[1], n, S));
        if (o1 > o0)
          copy_d2h_2d(st, const_cast<uint8_t*>(c.tape) + o0, c.tape_stride, rows.at(b0).tape + o0, rows.tape_stride, o1 - o0, Bc);
      }
      const double t_mid = ms_now();
      {
        const uint32_t kn = next_chunk.fetch_add(1);
        if (kn < nchunks) issue_inputs(kn, slot ^ 1);
        k = kn;
      }
      const uint32_t M = tot2[0];
      const size_t max_len = mode == 0 ? (size_t)proof_len((int)tot2[1], n, S)
                                       : (size_t)tot2[1] * REP0_LEN + (size_t)(S - (int)tot2[1]) * REP1_LEN;
      c.M = (int)M;
      c.item_b = w.take<uint32_t>(M);
      c.item_i = w.take<uint32_t>(M);
      c.item_k = w.take<uint32_t>(M);
      c.pb_T1 = w.take<uint32_t>((size_t)M * P256_PROJ_WORDS);
      c.pb_T1_aff = w.take<uint32_t>((size_t)M * 16);
      c.pb_T1_inf = w.take<uint8_t>(M);
      const size_t n2 = c.s2_count();
      c.s2_jv = w.take<uint32_t>(n2 * 8);
      c.s2_jr = w.take<uint32_t>(n2 * 8);
      c.s2_proj = w.take<uint32_t>(n2 * TOM_E2_WORDS);
      c.s2_aff = w.take<uint32_t>(n2 * TOM_AFF_WORDS);
      c.s2_bytes = w.take<uint8_t>(n2 * BSTRIDE);
      c.secrets = w.take<uint32_t>((size_t)M * SECRETS_PER_ITEM * 8);
      c.item_inv = w.take<uint32_t>((size_t)M * 8);
      c.item_chal = w.take<uint32_t>((size_t)M * HASHES_PER_ITEM * 3);
      c.gk_part = w.take_if<uint32_t>(gk_blocks(n) > 1, (size_t)Bc * n * gk_blocks(n) * 8);
      uint32_t* gext = w.take<uint32_t>(prove_gext_words(c));
      launch(st, Bc, ItemsTask{c});
      // --- phase B
      launch(st, M, PhaseBP256Task{c});
      launch_p256_norm(st, c.pb_T1, c.pb_T1_aff, nullptr, c.pb_T1_inf, (long long)(M));
      prove_items_gk(st, c, gext, true, true);
      launch(st, (long long)nA, RepEmitTask{c});
      if (mode == 0) launch(st, Bc, GkEmitTask{c});
      launch(st, (long long)Bc * FIN_PARTS, FinalizeTask{c});
      // --- self-check: k_b is the seed SeedProveTapeTask expanded, or the tape's first three draws
      if (check) {
        const uint8_t* key = seeded ? seeds : c.tape;
        check_chunk(ctx, P, ln, c, cin[slot], ring, ring_m, key, seeded ? 32 : c.tape_stride, seeded ? 32 : 96, b0, check_counts);
      }
      // --- results: on the output stream, behind this chunk's last kernel (its self-check included)
      ev_record(ln.ev_done[slot], st);
      if (ctx->progress && k_this < ctx->progress_cap) notify_progress(st, ctx->progress + k_this);
      if (!po.dev || !lo.dev || !so.dev) {
        Stream& co = ln.cs_out;
        ev_wait(co, ln.ev_done[slot]);
        // only the bytes up to the longest proof of the chunk are copied back (rows are stride-padded)
        // (one cudaMemcpyAsync per row with its exact length: 8192 driver calls per step cost more than
        // the ~25 % of padding they save)
        po.copy_back_2d(co, b0, c.proofs, Bc, max_len);
        lo.copy_back(co, b0, c.proof_len, Bc);
        so.copy_back(co, b0, c.status, Bc);
        ev_record(ln.ev_out[slot], co);
      }
      if (trace) {
        const double t_enq = ms_now();
        sync(st);
        const double t_comp = ms_now();
        sync(ln.cs_out);
        fprintf(stderr, "TRACE lane %d chunk %u rows %d begin %.2f mid %.2f enqueued %.2f computed %.2f copied %.2f\n", li, k_this, Bc,
                t_begin, t_mid, t_enq, t_comp, ms_now());
      }
    }
    uint32_t counts[2] = {0, 0};
    if (check) copy_d2h(st, counts, check_counts, sizeof(counts));
    sync(ln.cs_in);
    sync(ln.cs_out);
    sync(st);
    if (check) {
      std::lock_guard<std::mutex> g(ctx->stat_mu);
      ctx->self_check_rows += counts[0];
      ctx->self_check_fail += counts[1];
    }
  };
  run_lanes(ctx, used, run_lane);
  return 0;
}

// Every batched prove call: its argument checks (strides against the deepest ring used), then its prove_impl pass
static int prove_batch(zka_ctx* ctx, const zka_params* P, uint32_t B, const ProveRows& rows, const RingSrc& ring, int mode) {
  if (!ctx || !P || !rows.pk || (!rows.tape && !rows.seeds && !rows.hedge) || !rows.proofs || !rows.proof_len || !rows.status) return ZKA_E_ARG;
  if (mode == 0 && (!rows.msg_hash || !rows.sig || !rows.which || !(ring.set ? (const void*)rows.ring_of : ring.ring))) return ZKA_E_ARG;
  if (mode == 1 && (!rows.base || !rows.s_in)) return ZKA_E_ARG;
  const int S = (int)P->sec_level;
  auto check = [&](int n) {
    if (rows.proof_stride < (mode == 0 ? (size_t)proof_len(S, n, S) : (size_t)S * REP0_LEN)) return fail(ctx, ZKA_E_ARG, "proof_stride < zka_proof_max_len");
    if (rows.tape && rows.tape_stride < (size_t)32 * (mode == 0 ? prove_draws(0, n, S) : draws_before_items(S))) return fail(ctx, ZKA_E_ARG, "tape_stride too small");
    return 0;
  };
  return ring_passes(ctx, ring, rows.ring_of, B, check, [&](const RingSrc& pass) { return prove_impl(ctx, P, B, rows, pass, mode); });
}

int zka_prove_batch(zka_ctx* ctx, const zka_params* P, uint32_t B, const uint8_t* msg_hash, const uint8_t* sig,
                    const uint8_t* pk, const uint32_t* which, const uint8_t* ring, uint32_t N, const uint8_t* tape,
                    size_t tape_stride, uint8_t* proofs, size_t proof_stride, uint32_t* proof_len_out,
                    int32_t* status) {
  ProveRows r(proofs, proof_stride, proof_len_out, status);
  r.msg_hash = msg_hash; r.sig = sig; r.pk = pk; r.which = which; r.tape = tape; r.tape_stride = tape_stride;
  return prove_batch(ctx, P, B, r, RingSrc::one(ring, N), 0);
}

int zka_prove_batch_seeded(zka_ctx* ctx, const zka_params* P, uint32_t B, const uint8_t* msg_hash, const uint8_t* sig,
                           const uint8_t* pk, const uint32_t* which, const uint8_t* ring, uint32_t N, const uint8_t* seeds,
                           uint8_t* proofs, size_t proof_stride, uint32_t* proof_len_out, int32_t* status) {
  ProveRows r(proofs, proof_stride, proof_len_out, status);
  r.msg_hash = msg_hash; r.sig = sig; r.pk = pk; r.which = which; r.seeds = seeds;
  return prove_batch(ctx, P, B, r, RingSrc::one(ring, N), 0);
}

int zka_prove_batch_rings(zka_ctx* ctx, const zka_params* P, const zka_rings* rings, const uint32_t* ring_of, uint32_t B,
                          const uint8_t* msg_hash, const uint8_t* sig, const uint8_t* pk, const uint32_t* which, const uint8_t* tape,
                          size_t tape_stride, uint8_t* proofs, size_t proof_stride, uint32_t* proof_len_out, int32_t* status) {
  ProveRows r(proofs, proof_stride, proof_len_out, status);
  r.msg_hash = msg_hash; r.sig = sig; r.pk = pk; r.which = which; r.ring_of = ring_of; r.tape = tape; r.tape_stride = tape_stride;
  return prove_batch(ctx, P, B, r, RingSrc::pass(rings, 0), 0);
}

int zka_prove_batch_rings_seeded(zka_ctx* ctx, const zka_params* P, const zka_rings* rings, const uint32_t* ring_of, uint32_t B,
                                 const uint8_t* msg_hash, const uint8_t* sig, const uint8_t* pk, const uint32_t* which,
                                 const uint8_t* seeds, uint8_t* proofs, size_t proof_stride, uint32_t* proof_len_out, int32_t* status) {
  ProveRows r(proofs, proof_stride, proof_len_out, status);
  r.msg_hash = msg_hash; r.sig = sig; r.pk = pk; r.which = which; r.ring_of = ring_of; r.seeds = seeds;
  return prove_batch(ctx, P, B, r, RingSrc::pass(rings, 0), 0);
}

// ---- hedged seeds: the seeded calls with each row's seed derived on the device (SeedHedgeTask, rule in zk_seed.cuh)
int zka_prove_batch_hedged(zka_ctx* ctx, const zka_params* P, uint32_t B, const uint8_t* msg_hash, const uint8_t* sig,
                           const uint8_t* pk, const uint32_t* which, const uint8_t* ring, uint32_t N, const uint8_t* seeds,
                           uint8_t* proofs, size_t proof_stride, uint32_t* proof_len_out, int32_t* status) {
  ProveRows r(proofs, proof_stride, proof_len_out, status);
  r.msg_hash = msg_hash; r.sig = sig; r.pk = pk; r.which = which; r.seeds = seeds; r.hedge = true;
  return prove_batch(ctx, P, B, r, RingSrc::one(ring, N), 0);
}

int zka_prove_batch_rings_hedged(zka_ctx* ctx, const zka_params* P, const zka_rings* rings, const uint32_t* ring_of, uint32_t B,
                                 const uint8_t* msg_hash, const uint8_t* sig, const uint8_t* pk, const uint32_t* which,
                                 const uint8_t* seeds, uint8_t* proofs, size_t proof_stride, uint32_t* proof_len_out, int32_t* status) {
  ProveRows r(proofs, proof_stride, proof_len_out, status);
  r.msg_hash = msg_hash; r.sig = sig; r.pk = pk; r.which = which; r.ring_of = ring_of; r.seeds = seeds; r.hedge = true;
  return prove_batch(ctx, P, B, r, RingSrc::pass(rings, 0), 0);
}

// The seeds a hedged call derives, B x 32 into `out` (host or device, any alignment: the kernel writes a staging buffer),
// 1024 rows per launch
static int hedge_seeds(zka_ctx* ctx, const zka_params* P, uint32_t B, const ProveRows& rows, const RingSrc& ring, uint8_t* out) {
  if (!ctx || !P || !rows.msg_hash || !rows.sig || !rows.pk || !rows.which || !out) return ZKA_E_ARG;
  if (!(ring.set ? (const void*)rows.ring_of : ring.ring)) return ZKA_E_ARG;
  return ring_passes(ctx, ring, rows.ring_of, B, [](int) { return 0; }, [&](const RingSrc& pass) {
    Stream& st = ctx->st;
    pass.prepare(ctx, false, true);
    const uint32_t rows_per = 1024;
    for (uint32_t b0 = 0; b0 < B; b0 += rows_per) {
      const uint32_t Bc = std::min(rows_per, B - b0);
      const ProveRows r = rows.at(b0), e = rows.at(b0 + Bc);
      Cursor in(ctx->in[0]), w(ctx->w);
      auto stage = [&](auto* p, auto* end) { return stage_in(st, in.next(), p, (size_t)(end - p)); };
      SeedHedgeTask ht{{}, pass.digests(ctx), stage(r.ring_of, e.ring_of), stage(r.seeds, e.seeds), stage(r.msg_hash, e.msg_hash),
                       stage(r.sig, e.sig), stage(r.pk, e.pk), stage(r.which, e.which), w.take<uint8_t>((size_t)Bc * 32)};
      memcpy(ht.params_digest, P->hedge_digest, 32);
      launch(st, Bc, ht);
      copy_d2h(st, out + (size_t)b0 * 32, ht.out, (size_t)Bc * 32);   // (cudaMemcpyDefault: host or device)
      sync(st);
    }
    return 0;
  });
}

int zka_hedge_seeds(zka_ctx* ctx, const zka_params* P, uint32_t B, const uint8_t* msg_hash, const uint8_t* sig, const uint8_t* pk,
                    const uint32_t* which, const uint8_t* ring, uint32_t N, const uint8_t* seeds, uint8_t* out) {
  ProveRows r;
  r.msg_hash = msg_hash; r.sig = sig; r.pk = pk; r.which = which; r.seeds = seeds;
  return hedge_seeds(ctx, P, B, r, RingSrc::one(ring, N), out);
}

int zka_hedge_seeds_rings(zka_ctx* ctx, const zka_params* P, const zka_rings* rings, const uint32_t* ring_of, uint32_t B,
                          const uint8_t* msg_hash, const uint8_t* sig, const uint8_t* pk, const uint32_t* which, const uint8_t* seeds,
                          uint8_t* out) {
  ProveRows r;
  r.msg_hash = msg_hash; r.sig = sig; r.pk = pk; r.which = which; r.ring_of = ring_of; r.seeds = seeds;
  return hedge_seeds(ctx, P, B, r, RingSrc::pass(rings, 0), out);
}

// The tape a seed stands for (the rule of zk_seed.cuh): kind 0 all prove_draws(S, n, S) prover draws, kind 1 the verify
// layout for `samples`.  Rows are expanded into a 16-byte aligned staging buffer and copied out at the caller's stride.
int zka_seed_tape(zka_ctx* ctx, int kind, uint32_t B, const uint8_t* seeds, uint32_t ring_size, uint32_t sec_level,
                  uint32_t samples, uint8_t* tape, size_t tape_stride) {
  if (!ctx || !seeds || !tape || (kind != 0 && kind != 1)) return ZKA_E_ARG;
  if (B == 0) return 0;
  if (ring_size < 2 || ring_size > (1u << 20)) return fail(ctx, ZKA_E_ARG, "ring size must be in [2, 2^20]");
  if (sec_level < 1 || sec_level > MAX_REPS) return fail(ctx, ZKA_E_ARG, "sec_level must be in [1,80]");
  const int S = (int)sec_level, n = ceil_log2(ring_size), K = (int)samples;
  if (kind == 1 && K < 1) return fail(ctx, ZKA_E_ARG, "samples must be >= 1");
  if (kind == 1 && S < K) return fail(ctx, ZKA_E_ARG, "security level not achieved");
  const size_t len = kind == 0 ? (size_t)32 * prove_draws(S, n, S) : verify_tape_len(n, S, K);   // both multiples of 16
  if (tape_stride < len) return fail(ctx, ZKA_E_ARG, kind == 0 ? "tape_stride < zka_prove_tape_len" : "tape_stride < zka_verify_tape_len");
  return guarded(ctx, [&] {
    Stream& st = ctx->st;
    const uint32_t rows = 1024;
    for (uint32_t b0 = 0; b0 < B; b0 += rows) {
      const uint32_t Bc = std::min(rows, B - b0);
      Cursor in(ctx->in[0]), w(ctx->w);
      const uint8_t* ds = stage_in(st, in.next(), seeds + (size_t)b0 * 32, (size_t)Bc * 32);
      uint8_t* dt = w.take<uint8_t>((size_t)Bc * len);
      if (kind == 0) {
        launch(st, (long long)Bc * prove_draws(S, n, S), SeedProveTapeTask{ds, dt, len, S, n, 0, prove_draws(S, n, S), nullptr});
      } else {
        const SeedVerifyTapeTask vt{ds, dt, len, n, S, K};
        launch(st, (long long)Bc * vt.slots(), vt);
      }
      copy_d2h_2d(st, tape + (size_t)b0 * tape_stride, tape_stride, dt, len, len, Bc);
      sync(st);
    }
    return 0;
  });
}

// proveExp(paramsNIST = (p256, base, NistGroup.h), paramsWario = ProofGroup, s, Cs, P = pk, Px, Py, secparam = sec_level, Q?)
// (exp.ts:126-231).  Tape layout = zka_prove_batch's: draws 0..2 are the blinders of Cs, Px, Py (drawn when those
// commitments were made), then 4 per repetition, then 40 per 0-bit repetition.  Rows: the repetitions only.
int zka_prove_exp_batch(zka_ctx* ctx, const zka_params* P, uint32_t B, const uint8_t* base, const uint8_t* s, const uint8_t* pk,
                        const uint8_t* q, const uint8_t* tape, size_t tape_stride, uint8_t* proofs, size_t proof_stride,
                        uint32_t* proof_len, int32_t* status) {
  ProveRows r(proofs, proof_stride, proof_len, status);
  r.base = base; r.s_in = s; r.pk = pk; r.q_in = q; r.tape = tape; r.tape_stride = tape_stride;
  return prove_batch(ctx, P, B, r, RingSrc::none(0), 1);
}

// proveMembership(params = ProofGroup, com, index, ring) (gk.ts:94-195) for B commitments over one ring.
// com_r: the blinder of com = commit(ring[index]) (B x 32); tape: the 5n draws (r_i, a_i, s_i, t_i, rho_i per round).
// Rows: the GK block of the flat layout.
int zka_prove_membership_batch(zka_ctx* ctx, const zka_params* P, uint32_t B, const uint8_t* com_r, const uint32_t* index,
                               const uint8_t* ring, uint32_t N, const uint8_t* tape, size_t tape_stride, uint8_t* proofs,
                               size_t proof_stride, uint32_t* proof_len, int32_t* status) {
  if (!ctx || !P || !com_r || !index || !ring || !tape || !proofs || !proof_len || !status) return ZKA_E_ARG;
  if (B == 0) return 0;
  if (N < 2 || N > (1u << 20)) return fail(ctx, ZKA_E_ARG, "ring size must be in [2, 2^20]");
  const int n = ceil_log2(N);
  if (proof_stride < (size_t)gk_len(n)) return fail(ctx, ZKA_E_ARG, "proof_stride < GK block length");
  if (tape_stride < (size_t)32 * 5 * n) return fail(ctx, ZKA_E_ARG, "tape_stride < 32 * 5n");
  return guarded(ctx, [&] {
    Stream& st = ctx->st;
    const uint32_t* ring_m = prep_ring(ctx, st, ring, N, n, true);
    const Output<uint8_t> po(proofs, proof_stride);
    const Output<uint32_t> lo(proof_len, 1);
    const Output<int32_t> so(status, 1);
    // internal tape: [pad, com.r, pad] then the caller's draws (S = 0: GK draws start at 3); the row pitch is rounded up
    // to a multiple of 16 so that every draw is read with 16-byte loads
    const size_t it_len = 96 + tape_stride, it_stride = (it_len + 15) & ~(size_t)15;
    const uint32_t chunk = 8192;
    for (uint32_t b0 = 0; b0 < B; b0 += chunk) {
      const int Bc = (int)std::min<uint32_t>(chunk, B - b0);
      Cursor in(ctx->in[0]), w(ctx->w), ob(ctx->out[0]);
      const uint8_t* d_cr = stage_in(st, in.next(), com_r + (size_t)b0 * 32, (size_t)Bc * 32);
      const uint32_t* d_idx = stage_in(st, in.next(), index + b0, (size_t)Bc);
      const uint8_t* d_tape = stage_in(st, in.next(), tape + (size_t)b0 * tape_stride, (size_t)Bc * tape_stride);
      ProveCtx c = prove_ctx(ctx, P, Bc, 0, (int)N, n);
      c.which = d_idx;
      c.ring_m = ring_m;
      uint8_t* itape = w.take<uint8_t>((size_t)Bc * it_stride);
      c.tape = itape; c.tape_stride = it_stride; c.tape_draws = (uint32_t)(it_len / 32);
      c.which_s = w.take<uint32_t>(Bc);
      c.zcount = w.take<uint32_t>(Bc);
      c.gk_off = w.take<uint32_t>(Bc);
      c.gk_dv = w.take<uint32_t>((size_t)Bc * n * 8);
      c.gk_x = w.take<uint32_t>((size_t)Bc * 3);
      const size_t ng = (size_t)Bc * 4 * n;
      c.s2_jv = w.take<uint32_t>(ng * 8);
      c.s2_jr = w.take<uint32_t>(ng * 8);
      c.s2_proj = w.take<uint32_t>(ng * TOM_E2_WORDS);
      c.s2_bytes = w.take<uint8_t>(ng * BSTRIDE);
      c.gk_part = w.take_if<uint32_t>(gk_blocks(n) > 1, (size_t)Bc * n * gk_blocks(n) * 8);
      c.proof_stride = proof_stride;
      c.proofs = po.rows(ob.next(), b0, Bc);
      c.proof_len = lo.rows(ob.next(), b0, Bc);
      c.status = so.rows(ob.next(), b0, Bc);
      uint32_t* gext = w.take<uint32_t>(prove_gext_words(c));
      launch(st, Bc, GkAloneSetupTask{c, d_cr, d_tape, tape_stride, itape});
      prove_items_gk(st, c, gext, false, true);
      launch(st, Bc, GkEmitTask{c});
      launch(st, (long long)Bc * FIN_PARTS, FinalizeTask{c});
      po.copy_back_2d(st, b0, c.proofs, Bc, (size_t)gk_len(n));
      lo.copy_back(st, b0, c.proof_len, Bc);
      so.copy_back(st, b0, c.status, Bc);
      sync(st);
    }
    return 0;
  });
}

// proveEquality / proveMult alone (kind 0 / 1): see SubProveJobsTask
static int prove_sub(zka_ctx* ctx, const zka_params* P, int kind, uint32_t B, const uint8_t* scalars, const uint8_t* tape,
                     size_t tape_stride, uint8_t* commitments, uint8_t* proofs, int32_t* status) {
  if (!ctx || !P || !scalars || !tape || !commitments || !proofs || !status) return ZKA_E_ARG;
  if (B == 0) return 0;
  const int ns = kind == 0 ? 3 : 6, nd = kind == 0 ? 3 : 7, J = kind == 0 ? SUBP_EQ_JOBS : SUBP_MULT_JOBS;
  const int nc = kind == 0 ? 2 : 3, plen = kind == 0 ? EQ_LEN : MULT_LEN;
  if (tape_stride < (size_t)32 * nd) return fail(ctx, ZKA_E_ARG, "tape_stride too small for this sub-proof");
  return guarded(ctx, [&] {
    Stream& st = ctx->st;
    const Output<uint8_t> co(commitments, (size_t)nc * WP), po(proofs, plen);
    const Output<int32_t> so(status, 1);
    const uint32_t chunk = 16384;
    for (uint32_t b0 = 0; b0 < B; b0 += chunk) {
      const int Bc = (int)std::min<uint32_t>(chunk, B - b0);
      Cursor in(ctx->in[0]), w(ctx->w), ob(ctx->out[0]);
      const uint8_t* d_sc = stage_in(st, in.next(), scalars + (size_t)b0 * ns * 32, (size_t)Bc * ns * 32);
      const uint8_t* d_tape = stage_in(st, in.next(), tape + (size_t)b0 * tape_stride, (size_t)Bc * tape_stride);
      const size_t nj = (size_t)Bc * J;
      uint32_t* jv = w.take<uint32_t>(nj * 8);
      uint32_t* jr = w.take<uint32_t>(nj * 8);
      uint32_t* proj = w.take<uint32_t>(nj * TOM_E2_WORDS);
      uint8_t* bytes = w.take<uint8_t>(nj * BSTRIDE);
      uint8_t* d_com = co.rows(ob.next(), b0, Bc);
      uint8_t* d_prf = po.rows(ob.next(), b0, Bc);
      int32_t* d_st = so.rows(ob.next(), b0, Bc);
      launch(st, Bc, SubProveJobsTask{kind, d_sc, d_tape, tape_stride, jv, jr, d_st});
      launch(st, (long long)nj, TomCommitTask{jv, jr, ctx->tg.tab, P->th.tab, proj, ctx->tom});
      launch_tom_norm(st, proj, nullptr, bytes, (long long)nj, 1);
      launch(st, Bc, SubProveEmitTask{kind, d_sc, d_tape, tape_stride, jr, bytes, d_com, d_prf, d_st});
      co.copy_back(st, b0, d_com, Bc);
      po.copy_back(st, b0, d_prf, Bc);
      so.copy_back(st, b0, d_st, Bc);
      sync(st);
    }
    return 0;
  });
}
int zka_prove_equality_batch(zka_ctx* ctx, const zka_params* P, uint32_t B, const uint8_t* scalars, const uint8_t* tape,
                             size_t tape_stride, uint8_t* commitments, uint8_t* proofs, int32_t* status) {
  return prove_sub(ctx, P, 0, B, scalars, tape, tape_stride, commitments, proofs, status);
}
int zka_prove_mult_batch(zka_ctx* ctx, const zka_params* P, uint32_t B, const uint8_t* scalars, const uint8_t* tape,
                         size_t tape_stride, uint8_t* commitments, uint8_t* proofs, int32_t* status) {
  return prove_sub(ctx, P, 1, B, scalars, tape, tape_stride, commitments, proofs, status);
}

// provePointAdd alone (pointAdd.ts:92-163): the item stages of the batched prover with S = 1 (see PaddSetupTask)
int zka_prove_pointadd_batch(zka_ctx* ctx, const zka_params* P, uint32_t B, const uint8_t* points, const uint8_t* blinders,
                             const uint8_t* tape, size_t tape_stride, uint8_t* commitments, uint8_t* proofs, int32_t* status) {
  if (!ctx || !P || !points || !blinders || !tape || !commitments || !proofs || !status) return ZKA_E_ARG;
  if (B == 0) return 0;
  if (tape_stride < (size_t)32 * 38) return fail(ctx, ZKA_E_ARG, "tape_stride < 32 * 38");
  return guarded(ctx, [&] {
    Stream& st = ctx->st;
    const size_t it_stride = (size_t)32 * (9 + 38);   // a multiple of 16: every draw is read with 16-byte loads
    const size_t row_stride = REP0_LEN;
    const Output<uint8_t> co(commitments, 6 * WP), po(proofs, PA_LEN);
    const Output<int32_t> so(status, 1);
    const uint32_t chunk = 8192;
    for (uint32_t b0 = 0; b0 < B; b0 += chunk) {
      const int Bc = (int)std::min<uint32_t>(chunk, B - b0);
      Cursor in(ctx->in[0]), w(ctx->w), ob(ctx->out[0]);
      const uint8_t* d_pts = stage_in(st, in.next(), points + (size_t)b0 * 195, (size_t)Bc * 195);
      const uint8_t* d_bl = stage_in(st, in.next(), blinders + (size_t)b0 * 192, (size_t)Bc * 192);
      const uint8_t* d_tape = stage_in(st, in.next(), tape + (size_t)b0 * tape_stride, (size_t)Bc * tape_stride);
      ProveCtx c = prove_ctx(ctx, P, Bc, 1, 2, 0);
      c.M = Bc; c.mode = 1; c.head_len = 0;
      uint8_t* itape = w.take<uint8_t>((size_t)Bc * it_stride);
      c.tape = itape; c.tape_stride = it_stride; c.tape_draws = (uint32_t)(it_stride / 32);
      const size_t n1 = (size_t)Bc * 4, n2 = (size_t)Bc * (JOBS_PER_ITEM + DERS_PER_ITEM);
      c.s1 = w.take<uint32_t>((size_t)Bc * 8);
      c.pk_aff = w.take<uint32_t>((size_t)Bc * 16);
      c.pa_T_aff = w.take<uint32_t>((size_t)Bc * 2 * 16);
      c.pa_T_inf = w.take<uint8_t>((size_t)Bc * 2);
      c.pa_A_inf = w.take<uint8_t>((size_t)Bc * 2);
      c.pb_T1_aff = w.take<uint32_t>((size_t)Bc * 16);
      c.pb_T1_inf = w.take<uint8_t>(Bc);
      c.chal = w.take<uint32_t>((size_t)Bc * 3);
      c.zcount = w.take<uint32_t>(Bc);
      c.item_base = w.take<uint32_t>(Bc);
      c.item_b = w.take<uint32_t>(Bc);
      c.item_i = w.take<uint32_t>(Bc);
      c.item_k = w.take<uint32_t>(Bc);
      c.rep_off = w.take<uint32_t>(Bc);
      c.s1_jv = w.take<uint32_t>(n1 * 8);
      c.s1_jr = w.take<uint32_t>(n1 * 8);
      c.s1_proj = w.take<uint32_t>(n1 * TOM_E2_WORDS);
      c.s1_aff = w.take<uint32_t>(n1 * TOM_AFF_WORDS);
      c.s1_bytes = w.take<uint8_t>(n1 * BSTRIDE);
      c.s2_jv = w.take<uint32_t>(n2 * 8);
      c.s2_jr = w.take<uint32_t>(n2 * 8);
      c.s2_proj = w.take<uint32_t>(n2 * TOM_E2_WORDS);
      c.s2_aff = w.take<uint32_t>(n2 * TOM_AFF_WORDS);
      c.s2_bytes = w.take<uint8_t>(n2 * BSTRIDE);
      c.secrets = w.take<uint32_t>((size_t)Bc * SECRETS_PER_ITEM * 8);
      c.item_inv = w.take<uint32_t>((size_t)Bc * 8);
      c.item_chal = w.take<uint32_t>((size_t)Bc * HASHES_PER_ITEM * 3);
      uint32_t* gext = w.take<uint32_t>(prove_gext_words(c));
      c.proof_stride = row_stride;
      c.proofs = w.take<uint8_t>((size_t)Bc * row_stride);
      c.proof_len = w.take<uint32_t>(Bc);
      uint8_t* d_com = co.rows(ob.next(), b0, Bc);
      uint8_t* d_prf = po.rows(ob.next(), b0, Bc);
      c.status = so.rows(ob.next(), b0, Bc);
      launch(st, Bc, PaddSetupTask{c, d_pts, d_bl, d_tape, tape_stride, itape});
      prove_store1(st, c);
      prove_items_gk(st, c, gext, true, false);
      launch(st, Bc, PaddExtractTask{c, d_com, d_prf});
      co.copy_back(st, b0, d_com, Bc);
      po.copy_back(st, b0, d_prf, Bc);
      so.copy_back(st, b0, c.status, Bc);
      sync(st);
    }
    return 0;
  });
}

size_t zka_verify_tape_len_ex(uint32_t ring_size, uint32_t sec_level, uint32_t samples) {
  return verify_tape_len(ceil_log2(ring_size), (int)sec_level, (int)samples);
}

// mode 0: verifySignatureList; mode 1: verifyExp alone on assembled rows (msg_hash unused, Q from q_ext)
// seeds (B x 32, mode 0 only) instead of a tape: SeedVerifyTapeTask expands each chunk's verify layout on the lane's stream
static int verify_impl(zka_ctx* ctx, const zka_params* P, uint32_t B, const VerifyRows& rows, const RingSrc& ring,
                       uint32_t samples, int mode) {
  const int S = (int)P->sec_level, K = (int)samples, n = ring.n;
  const bool seeded = rows.seeds != nullptr;
  const size_t seed_stride = verify_tape_len(n, S, K);   // a multiple of 16
  const uint32_t* ring_m = ring.prepare(ctx, false);
  const Output<uint8_t> oo(rows.ok, 1);
  const Output<int32_t> so(rows.status, 1);
  const int lanes = ctx->nlanes;
  const bool all_dev = is_device_ptr(rows.proofs) && is_device_ptr(seeded ? rows.seeds : rows.tape);
  // (two equal chunks per lane instead of the tapered host schedule: no gain at batch 8192, slower at batch 1024)
  const std::vector<uint32_t> off = chunk_schedule(B, (uint32_t)std::min(ctx->chunk, all_dev ? 4096 : std::min(4096, ctx->host_chunk)), lanes, !all_dev);
  const uint32_t nchunks = (uint32_t)off.size() - 1;
  const int used = (int)std::min<uint32_t>((uint32_t)lanes, nchunks);
  std::atomic<uint32_t> next_chunk((uint32_t)used);
  const bool trace = getenv("ZKA_TRACE") != nullptr;
  const auto t_call = std::chrono::steady_clock::now();
  auto ms_now = [&] { return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t_call).count(); };
  // every lane starts with chunk `li` and then claims chunks from a shared counter: copy-in, kernels and copy-out of a chunk are sequential on the
  // lane's stream; the copies of one lane overlap the kernels of the others
  // the inputs of a lane's NEXT chunk travel on the copy-in stream (second set of staging buffers) while the current
  // chunk computes; a chunk's kernels wait for its event only
  auto stage_chunk = [&](Lane& ln, int slot, uint32_t kk) {
    // ONE copy-in stream for all lanes of the call: the chunks' inputs cross PCIe in the order they were queued, each at
    // full bandwidth (with a copy stream per lane the first chunks and the prefetched ones were all in flight at once).
    std::lock_guard<std::mutex> copy_lock(ctx->copy_mu);
    Stream& ci = ctx->cs_in;
    Cursor in(ln.in[slot]);
    DevBuf& rows_buf = in.next();   // first, like the prover's tape: the largest inputs share one buffer
    // the chunk's rows of an input: from its first row to the next chunk's (q_ext is device memory already)
    const VerifyRows r = rows.at(off[kk]), e = rows.at(off[kk + 1]);
    const size_t Bc = off[kk + 1] - off[kk], proof_stride = rows.proof_stride;
    auto stage = [&](auto* p, auto* end) { return stage_in(ci, in.next(), p, (size_t)(end - p)); };
    VerifyRows v = r;
    v.msg_hash = stage(r.msg_hash, e.msg_hash);
    if (is_device_ptr(rows.proofs) || is_device_ptr(rows.proof_len)) {
      v.proofs = stage_in(ci, rows_buf, r.proofs, (size_t)(e.proofs - r.proofs));
    } else {
      // host rows: only the bytes up to the longest proof of the chunk cross PCIe (rows are stride-padded;
      // a length above the stride is rejected by VLayoutTask without reading the row)
      size_t w = 0;
      for (size_t i = 0; i < Bc; i++) w = std::max<size_t>(w, r.proof_len[i]);
      w = std::min(proof_stride, (w + 15) & ~(size_t)15);
      uint8_t* dp = rows_buf.get<uint8_t>(Bc * proof_stride);
      copy_d2h_2d(ci, dp, proof_stride, r.proofs, proof_stride, w, Bc);
      v.proofs = dp;
    }
    v.proof_len = stage(r.proof_len, e.proof_len);
    if (seeded) v.tape = in.next().get<uint8_t>(Bc * seed_stride);   // filled by SeedVerifyTapeTask
    else v.tape = stage(r.tape, e.tape);
    v.seeds = stage(r.seeds, e.seeds);
    v.ring_of = stage(r.ring_of, e.ring_of);
    ev_record(ln.ev_small[slot], ci);
    return v;
  };
  // the first chunk of every lane is queued here, in chunk order, before any lane prefetches its second one (otherwise a
  // lane queues its first chunk and its prefetch back to back, and another lane's first inputs land late)
  std::vector<VerifyRows> first((size_t)used);
  for (int li = 0; li < used; li++) first[(size_t)li] = stage_chunk(ctx->lane(li), 0, (uint32_t)li);
  auto run_lane = [&](int li) {
    Lane& ln = ctx->lane(li);
    Stream& st = ln.st;
    uint32_t k = (uint32_t)li;
    if (k >= nchunks) return;
    int slot = 0;
    VerifyRows cur = first[(size_t)li];
    for (;;) {
    // claim the next chunk now and send its inputs on their way (the other slot's buffers were last read by the chunk
    // before this one, which ended with a stream synchronisation)
    const uint32_t kn = next_chunk.fetch_add(1);
    VerifyRows nxt{};
    if (kn < nchunks) nxt = stage_chunk(ln, slot ^ 1, kn);
    ev_wait(st, ln.ev_small[slot]);
    const uint32_t b0 = off[k];
    const int Bc = (int)(off[k + 1] - b0);
    const double t_begin = trace ? ms_now() : 0.0;
    VerifyCtx c = verify_ctx(ctx, P, Bc, S, (int)ring.N, n, K, mode);
    c.q_ext = cur.q_ext;
    c.msg_hash = cur.msg_hash;
    c.proofs = cur.proofs;
    c.proof_stride = rows.proof_stride;
    c.proof_len = cur.proof_len;
    c.tape = cur.tape;
    c.tape_stride = seeded ? seed_stride : rows.tape_stride;
    ring.fill(c, ring_m, cur.ring_of);
    if (seeded) {
      const SeedVerifyTapeTask vt{cur.seeds, const_cast<uint8_t*>(cur.tape), seed_stride, n, S, K, c.ring_of, c.ring_depth};
      launch(st, (long long)Bc * vt.slots(), vt);
    }
    double t_in = 0.0;
    if (trace) { sync(st); t_in = ms_now(); }
    Cursor ob(ln.out[0]);
    c.ok = oo.rows(ob.next(), b0, Bc);
    c.status = so.rows(ob.next(), b0, Bc);
    const uint32_t* ctl = verify_chunk(ctx, ln, c, b0, ctx->agg && mode == 0, &ctx->agg_c_last);
    oo.copy_back(st, b0, c.ok, Bc);
    so.copy_back(st, b0, c.status, Bc);
    uint32_t hctl[AGG_CTL_WORDS] = {0, 0, 0, 0};
    if (ctl) copy_d2h(st, hctl, ctl, sizeof(hctl));
    const double t_enq = trace ? ms_now() : 0.0;
    sync(st);
    if (trace)
      fprintf(stderr, "VTRACE lane %d chunk %u rows %d begin %.2f inputs_on_device %.2f enqueued %.2f done %.2f\n", li, k, Bc, t_begin, t_in,
              t_enq, ms_now());
    if (ctl) {
      std::lock_guard<std::mutex> g(ctx->stat_mu);
      if (hctl[AGG_TOM_PASS] && hctl[AGG_NIST_PASS]) ctx->agg_pass++;
      else ctx->agg_fail++;
    }
    if (kn >= nchunks) break;
    k = kn;
    cur = nxt;
    slot ^= 1;
  }
  };
  run_lanes(ctx, used, run_lane);
  sync(ctx->cs_in);
  return 0;
}

// Every batched verify call: its argument checks (tape stride against the deepest ring used), then its verify_impl pass
static int verify_batch(zka_ctx* ctx, const zka_params* P, uint32_t B, const VerifyRows& rows, const RingSrc& ring,
                        uint32_t samples, int mode) {
  if (!ctx || !P || !rows.proofs || !rows.proof_len || (!rows.tape && !rows.seeds) || !rows.ok || !rows.status) return ZKA_E_ARG;
  if (mode == 0 && (!rows.msg_hash || !(ring.set ? (const void*)rows.ring_of : ring.ring))) return ZKA_E_ARG;
  const int S = (int)P->sec_level, K = (int)samples;
  auto check = [&](int n) {
    if (K < 1) return fail(ctx, ZKA_E_ARG, "samples must be >= 1");
    // verifyExp throws 'security level not achieved' when secparam > pi.length (exp.ts:243-245)
    if (S < K) return fail(ctx, ZKA_E_ARG, "security level not achieved");
    if (rows.tape && rows.tape_stride < (mode == 1 ? (size_t)V_IDX_PAD + (size_t)32 * 25 * K : verify_tape_len(n, S, K)))
      return fail(ctx, ZKA_E_ARG, "tape_stride < zka_verify_tape_len");
    return 0;
  };
  return ring_passes(ctx, ring, rows.ring_of, B, check, [&](const RingSrc& pass) { return verify_impl(ctx, P, B, rows, pass, samples, mode); });
}

int zka_verify_batch(zka_ctx* ctx, const zka_params* P, uint32_t B, const uint8_t* msg_hash, const uint8_t* ring,
                     uint32_t N, const uint8_t* proofs, size_t proof_stride, const uint32_t* proof_len,
                     const uint8_t* tape, size_t tape_stride, uint8_t* ok, int32_t* status) {
  // verifySignatureList hard-codes secparam = 20 (zkpAttestList.ts:177)
  return zka_verify_batch_ex(ctx, P, B, msg_hash, ring, N, proofs, proof_stride, proof_len, tape, tape_stride, ok, status, V_SAMPLES);
}

int zka_verify_batch_ex(zka_ctx* ctx, const zka_params* P, uint32_t B, const uint8_t* msg_hash, const uint8_t* ring,
                        uint32_t N, const uint8_t* proofs, size_t proof_stride, const uint32_t* proof_len,
                        const uint8_t* tape, size_t tape_stride, uint8_t* ok, int32_t* status, uint32_t samples) {
  VerifyRows r(proofs, proof_stride, proof_len, ok, status);
  r.msg_hash = msg_hash; r.tape = tape; r.tape_stride = tape_stride;
  return verify_batch(ctx, P, B, r, RingSrc::one(ring, N), samples, 0);
}

int zka_verify_batch_seeded(zka_ctx* ctx, const zka_params* P, uint32_t B, const uint8_t* msg_hash, const uint8_t* ring,
                            uint32_t N, const uint8_t* proofs, size_t proof_stride, const uint32_t* proof_len,
                            const uint8_t* seeds, uint32_t samples, uint8_t* ok, int32_t* status) {
  VerifyRows r(proofs, proof_stride, proof_len, ok, status);
  r.msg_hash = msg_hash; r.seeds = seeds;
  return verify_batch(ctx, P, B, r, RingSrc::one(ring, N), samples, 0);
}

int zka_verify_batch_rings(zka_ctx* ctx, const zka_params* P, const zka_rings* rings, const uint32_t* ring_of, uint32_t B,
                           const uint8_t* msg_hash, const uint8_t* proofs, size_t proof_stride, const uint32_t* proof_len,
                           const uint8_t* tape, size_t tape_stride, uint32_t samples, uint8_t* ok, int32_t* status) {
  VerifyRows r(proofs, proof_stride, proof_len, ok, status);
  r.msg_hash = msg_hash; r.ring_of = ring_of; r.tape = tape; r.tape_stride = tape_stride;
  return verify_batch(ctx, P, B, r, RingSrc::pass(rings, 0), samples, 0);
}

int zka_verify_batch_rings_seeded(zka_ctx* ctx, const zka_params* P, const zka_rings* rings, const uint32_t* ring_of, uint32_t B,
                                  const uint8_t* msg_hash, const uint8_t* proofs, size_t proof_stride, const uint32_t* proof_len,
                                  const uint8_t* seeds, uint32_t samples, uint8_t* ok, int32_t* status) {
  VerifyRows r(proofs, proof_stride, proof_len, ok, status);
  r.msg_hash = msg_hash; r.ring_of = ring_of; r.seeds = seeds;
  return verify_batch(ctx, P, B, r, RingSrc::pass(rings, 0), samples, 0);
}

// ------------------------------------------------------------------ stand-alone sub-proof verifiers
// verifyExp(paramsNIST = (p256, base, NistGroup.h), paramsWario = ProofGroup, Clambda, Px, Py, pi, secparam, Q?)
// (exp.ts:233-349) for B independent statements.  The repetitions arrive in the flat layout of include/zkattest.h.
int zka_verify_exp_batch(zka_ctx* ctx, const zka_params* P, uint32_t B, const uint8_t* base, const uint8_t* com,
                         const uint8_t* px, const uint8_t* py, const uint8_t* q, const uint8_t* proofs, size_t proof_stride,
                         const uint32_t* proof_len, const uint8_t* tape, size_t tape_stride, uint32_t samples, uint8_t* ok,
                         int32_t* status) {
  if (!ctx || !P || !base || !com || !px || !py || !proofs || !proof_len || !tape || !ok || !status || proof_stride == 0) return ZKA_E_ARG;
  if (B == 0) return 0;
  return guarded(ctx, [&] {
    Stream& st = ctx->st;
    DevBuf bufs[10];   // not the lane's staging buffers: verify_batch stages through those
    Cursor in(bufs);
    const uint8_t* d_base = stage_in(st, in.next(), base, (size_t)B * NP);
    const uint8_t* d_com = stage_in(st, in.next(), com, (size_t)B * NP);
    const uint8_t* d_px = stage_in(st, in.next(), px, (size_t)B * WP);
    const uint8_t* d_py = stage_in(st, in.next(), py, (size_t)B * WP);
    const uint8_t* d_q = stage_in(st, in.next(), q, (size_t)B * NP);
    const uint8_t* d_body = stage_in(st, in.next(), proofs, (size_t)B * proof_stride);
    const uint32_t* d_len = stage_in(st, in.next(), proof_len, (size_t)B);
    const uint8_t* d_tape = stage_in(st, in.next(), tape, (size_t)B * tape_stride);
    const size_t row_stride = (HEAD_LEN + proof_stride + 15) & ~(size_t)15;
    uint8_t* d_rows = in.take<uint8_t>((size_t)B * row_stride);
    uint32_t* d_rlen = in.take<uint32_t>(B);
    const int pieces = (int)((row_stride + 63) / 64);
    launch(st, (long long)B * pieces, VAssembleTask{d_base, d_com, d_px, d_py, d_body, proof_stride, d_len, d_rows, row_stride, d_rlen, pieces});
    sync(st);
    VerifyRows r(d_rows, row_stride, d_rlen, ok, status);
    r.tape = d_tape; r.tape_stride = tape_stride; r.q_ext = d_q;
    // n = 1 sizes GK workspace (ngk = 4n + 1) that mode 1 never fills, keeping the lane pools' layout as it has been
    return verify_batch(ctx, P, B, r, RingSrc::none(1), samples, 1);
  });
}

// verifyMembership(ProofGroup params, com, ring, proof) (gk.ts:197-262) for B commitments over one ring.
// tape: the 2n+1 Relation.drain scalars per proof, in call order.
int zka_verify_membership_batch(zka_ctx* ctx, const zka_params* P, uint32_t B, const uint8_t* com, const uint8_t* ring, uint32_t N,
                                const uint8_t* proofs, size_t proof_stride, const uint32_t* proof_len, const uint8_t* tape,
                                size_t tape_stride, uint8_t* ok, int32_t* status) {
  if (!ctx || !P || !com || !ring || !proofs || !proof_len || !tape || !ok || !status || proof_stride == 0) return ZKA_E_ARG;
  if (B == 0) return 0;
  if (N < 2 || N > (1u << 20)) return fail(ctx, ZKA_E_ARG, "ring size must be in [2, 2^20]");
  const int n = ceil_log2(N);
  if (tape_stride < (size_t)32 * (2 * n + 1)) return fail(ctx, ZKA_E_ARG, "tape_stride < 32 * (2n + 1)");
  return guarded(ctx, [&] {
    Stream& st = ctx->st;
    DevBuf bufs[4];
    const uint32_t* ring_m = prep_ring(ctx, st, ring, N, n, false);
    const Output<uint8_t> oo(ok, 1);
    const Output<int32_t> so(status, 1);
    const size_t row_stride = (HEAD_LEN + proof_stride + 15) & ~(size_t)15;
    const int pieces = (int)((row_stride + 63) / 64);
    const int ngk = 4 * n + 1;
    const uint32_t chunk = 4096;
    for (uint32_t b0 = 0; b0 < B; b0 += chunk) {
      const int Bc = (int)std::min<uint32_t>(chunk, B - b0);
      Cursor in(bufs), w(ctx->w), ob(ctx->out[0]);
      const uint8_t* d_com = stage_in(st, in.next(), com + (size_t)b0 * WP, (size_t)Bc * WP);
      const uint8_t* d_body = stage_in(st, in.next(), proofs + (size_t)b0 * proof_stride, (size_t)Bc * proof_stride);
      const uint32_t* d_len = stage_in(st, in.next(), proof_len + b0, (size_t)Bc);
      VerifyCtx c = verify_ctx(ctx, P, Bc, (int)P->sec_level, (int)N, n, 1, 2);
      c.tape = stage_in(st, in.next(), tape + (size_t)b0 * tape_stride, (size_t)Bc * tape_stride);
      c.tape_stride = tape_stride;
      c.ring_m = ring_m;
      uint8_t* d_rows = w.take<uint8_t>((size_t)Bc * row_stride);
      uint32_t* d_rlen = w.take<uint32_t>(Bc);
      c.proofs = d_rows; c.proof_stride = row_stride; c.proof_len = d_rlen;
      c.gk_off = w.take<uint32_t>(Bc);
      c.gk_ok_len = w.take<uint8_t>(Bc);
      c.gk_scalar = w.take<uint32_t>((size_t)Bc * ngk * 8);
      c.gk_pre = w.take<uint32_t>((size_t)Bc * ngk * TOM_PRE_WORDS);
      uint32_t* gk_offs = w.take<uint32_t>((size_t)Bc * ngk);
      c.fx_jv = w.take<uint32_t>((size_t)Bc * 2 * 8);
      c.fx_jr = w.take<uint32_t>((size_t)Bc * 2 * 8);
      c.fx_proj = w.take<uint32_t>((size_t)Bc * 2 * TOM_PROJ_WORDS);
      c.win_g = w.take<uint32_t>((size_t)Bc * MSM_NWIN * 36);
      c.id_flags = w.take<uint8_t>((size_t)Bc * 3);
      c.gk_part = w.take_if<uint32_t>(gk_blocks(n) > 1, (size_t)Bc * gk_blocks(n) * 8);
      c.ok = oo.rows(ob.next(), b0, Bc);
      c.status = so.rows(ob.next(), b0, Bc);
      launch(st, (long long)Bc * pieces, VAssembleTask{nullptr, nullptr, d_com, nullptr, d_body, proof_stride, d_len, d_rows, row_stride, d_rlen, pieces});
      launch(st, Bc, VGkOnlyLayoutTask{c});
      dev_memset(st, c.fx_jv, 0, (size_t)Bc * 2 * 8 * 4);
      dev_memset(st, c.fx_jr, 0, (size_t)Bc * 2 * 8 * 4);
      verify_gk(st, c, gk_offs);
      launch(st, (long long)Bc * ngk, VParseEntriesTask{c.proofs, row_stride, gk_offs, c.gk_pre, ngk});
      launch(st, (long long)Bc * 2, TomCommitTask{c.fx_jv, c.fx_jr, c.tg_tab, c.th_tab, c.fx_proj, c.tom, 1});
      launch(st, (long long)Bc * MSM_NWIN, MsmTomWindowTask{c.gk_scalar, c.gk_pre, nullptr, ngk, 0, 0, ngk, V_SEG, 1, c.win_g});
      launch(st, Bc, MsmTomCombineTask{c.win_g, c.fx_proj, c.id_flags, 2, 0, 0});
      launch(st, Bc, VGkOnlyFinalTask{c});
      oo.copy_back(st, b0, c.ok, Bc);
      so.copy_back(st, b0, c.status, Bc);
      sync(st);
    }
    return 0;
  });
}

// verifyEquality / verifyMult / verifyPointAdd alone (kind = 0 / 1 / 2): fixed-size inputs and proofs
static int verify_sub(zka_ctx* ctx, const zka_params* P, int kind, uint32_t B, const uint8_t* points, const uint8_t* proofs,
                      const uint8_t* tape, size_t tape_stride, uint8_t* ok, int32_t* status) {
  if (!ctx || !P || !points || !proofs || !tape || !ok || !status) return ZKA_E_ARG;
  if (B == 0) return 0;
  if (tape_stride < (size_t)32 * sub_draws(kind)) return fail(ctx, ZKA_E_ARG, "tape_stride too small for this sub-proof");
  return guarded(ctx, [&] {
    Stream& st = ctx->st;
    const int la = sub_points(kind) * WP, lc = sub_proof_len(kind), ne = sub_entries(kind);
    const size_t stride = (size_t)(la + lc + 15) & ~(size_t)15;
    const Output<uint8_t> oo(ok, 1);
    const Output<int32_t> so(status, 1);
    const uint32_t chunk = 8192;
    for (uint32_t b0 = 0; b0 < B; b0 += chunk) {
      const int Bc = (int)std::min<uint32_t>(chunk, B - b0);
      Cursor in(ctx->in[0]), w(ctx->w), ob(ctx->out[0]);
      const uint8_t* d_pts = stage_in(st, in.next(), points + (size_t)b0 * la, (size_t)Bc * la);
      const uint8_t* d_prf = stage_in(st, in.next(), proofs + (size_t)b0 * lc, (size_t)Bc * lc);
      const uint8_t* d_tape = stage_in(st, in.next(), tape + (size_t)b0 * tape_stride, (size_t)Bc * tape_stride);
      uint8_t* rows = w.take<uint8_t>((size_t)Bc * stride);
      uint32_t* ent_scalar = w.take<uint32_t>((size_t)Bc * SUB_ENT_MAX * 8);
      uint32_t* ent_off = w.take<uint32_t>((size_t)Bc * SUB_ENT_MAX);
      uint32_t* ent_pre = w.take<uint32_t>((size_t)Bc * SUB_ENT_MAX * TOM_PRE_WORDS);
      uint32_t* fx_jv = w.take<uint32_t>((size_t)Bc * 2 * 8);
      uint32_t* fx_jr = w.take<uint32_t>((size_t)Bc * 2 * 8);
      uint32_t* fx_proj = w.take<uint32_t>((size_t)Bc * 2 * TOM_PROJ_WORDS);
      uint32_t* win = w.take<uint32_t>((size_t)Bc * MSM_NWIN * 36);
      uint8_t* flags = w.take<uint8_t>((size_t)Bc * 3);
      uint8_t* d_ok = oo.rows(ob.next(), b0, Bc);
      int32_t* d_st = so.rows(ob.next(), b0, Bc);
      launch(st, (long long)Bc * (la + lc), VConcatTask{d_pts, d_prf, la, lc, rows, stride});
      launch(st, Bc, VSubProofTask{kind, rows, stride, d_tape, tape_stride, (const uint8_t*)ctx->tg_bytes.p, ent_scalar, ent_off,
                                   fx_jv, fx_jr, d_st, d_ok});
      launch(st, (long long)Bc * SUB_ENT_MAX, VParseEntriesTask{rows, stride, ent_off, ent_pre, SUB_ENT_MAX});
      launch(st, (long long)Bc * 2, TomCommitTask{fx_jv, fx_jr, ctx->tg.tab, P->th.tab, fx_proj, ctx->tom, 1});
      launch(st, (long long)Bc * MSM_NWIN, MsmTomWindowTask{ent_scalar, ent_pre, nullptr, SUB_ENT_MAX, 0, 0, ne, V_SEG, 1, win});
      launch(st, Bc, MsmTomCombineTask{win, fx_proj, flags, 2, 1, 1});
      launch(st, Bc, VSubFinalTask{d_st, flags, d_ok});
      oo.copy_back(st, b0, d_ok, Bc);
      so.copy_back(st, b0, d_st, Bc);
      sync(st);
    }
    return 0;
  });
}
int zka_verify_equality_batch(zka_ctx* ctx, const zka_params* P, uint32_t B, const uint8_t* points, const uint8_t* proofs,
                              const uint8_t* tape, size_t tape_stride, uint8_t* ok, int32_t* status) {
  return verify_sub(ctx, P, SUB_EQ, B, points, proofs, tape, tape_stride, ok, status);
}
int zka_verify_mult_batch(zka_ctx* ctx, const zka_params* P, uint32_t B, const uint8_t* points, const uint8_t* proofs,
                          const uint8_t* tape, size_t tape_stride, uint8_t* ok, int32_t* status) {
  return verify_sub(ctx, P, SUB_MULT, B, points, proofs, tape, tape_stride, ok, status);
}
int zka_verify_pointadd_batch(zka_ctx* ctx, const zka_params* P, uint32_t B, const uint8_t* points, const uint8_t* proofs,
                              const uint8_t* tape, size_t tape_stride, uint8_t* ok, int32_t* status) {
  return verify_sub(ctx, P, SUB_PADD, B, points, proofs, tape, tape_stride, ok, status);
}

// ---------------------------------------------------------------------------- multi-GPU helpers
namespace {
int pack_common(zka_ctx* ctx, uint32_t B, uint8_t* rows, size_t stride, const uint32_t* len, uint8_t* packed, size_t cap,
                uint64_t* offsets, void* stream, int dir) {
  if (!ctx || !rows || !len || !packed || !offsets || stride == 0) return ZKA_E_ARG;
  if (B == 0) return 0;
#if !defined(ZKA_HOSTSIM)
  if (!is_device_ptr(rows) || !is_device_ptr(len) || !is_device_ptr(packed) || !is_device_ptr(offsets))
    return fail(ctx, ZKA_E_ARG, "zka_proofs_pack/unpack take device pointers");
#endif
  return guarded(ctx, [&] {
    Stream tmp;          // borrowed stream (not owned, never destroyed here); launch counters go to lane 0
    Stream* st = &ctx->st;
#if !defined(ZKA_HOSTSIM)
    if (stream) { tmp.s = (cudaStream_t)stream; st = &tmp; }
#endif
    const int pieces = (int)((stride + 15) / 16);
    launch(*st, 1, PackScanTask{len, offsets, (int)B});
    const bool al = (stride % 16 == 0) && (((size_t)rows | (size_t)packed) % 16 == 0);
    if (al) launch(*st, (long long)B * pieces, PackCopy16Task{rows, stride, len, offsets, packed, cap, pieces, dir});
    else launch(*st, (long long)B * pieces, PackCopyTask{rows, stride, len, offsets, packed, cap, pieces, dir});
    if (st == &tmp) ctx->st.launches += tmp.launches; else sync(*st);
    return 0;
  });
}
}  // namespace

int zka_proofs_pack(zka_ctx* ctx, uint32_t B, const uint8_t* proofs, size_t proof_stride, const uint32_t* proof_len,
                    uint8_t* packed, size_t cap, uint64_t* offsets, void* stream) {
  return pack_common(ctx, B, const_cast<uint8_t*>(proofs), proof_stride, proof_len, packed, cap, offsets, stream, 0);
}
int zka_proofs_unpack(zka_ctx* ctx, uint32_t B, const uint8_t* packed, size_t cap, const uint32_t* proof_len, uint8_t* proofs,
                      size_t proof_stride, uint64_t* offsets, void* stream) {
  return pack_common(ctx, B, proofs, proof_stride, proof_len, const_cast<uint8_t*>(packed), cap, offsets, stream, 1);
}


// ---------------------------------------------------------------------------- traceable proofs (zk_trace.cuh)
// The trace stages run on the context's stream after the untraced pass of the call, TRACE_CHUNK rows at a time (the
// prover: over the untraced call's own chunks, whose progress flags are raised once their blocks are in place).
namespace {
constexpr uint32_t TRACE_CHUNK = 4096;

// the opener key Y on the device when it parses as a point of the proof group, else null
const uint8_t* trace_y(zka_ctx* ctx, DevBuf& buf, const uint8_t* Y) {
  Stream& st = ctx->st;
  uint8_t* d = buf.get<uint8_t>(WP + 16);
  uint32_t* aff = reinterpret_cast<uint32_t*>(ctx->trace[0].get<uint32_t>(TOM_AFF_WORDS));
  copy_h2d(st, d, Y, WP);
  launch(st, 1, ParsePointsTask{nullptr, d, nullptr, aff, d + WP, nullptr});
  uint8_t bad = 1;
  copy_d2h(st, &bad, d + WP, 1);
  sync(st);
  return bad ? nullptr : d;
}
// sk (32 bytes big-endian, host or device) as limbs; false unless 1 <= sk < q
bool trace_sk(zka_ctx* ctx, const uint8_t* sk, uint32_t* out) {
  uint8_t h[32];
  copy_d2h(ctx->st, h, sk, 32);
  sync(ctx->st);
  limbs_from_be<8>(out, h, 32);
  return !is_zero_n<8>(out) && lt_p<FpP256>(out);
}
// the encoding of sk g on the device (BSTRIDE bytes)
uint8_t* trace_pubkey_dev(zka_ctx* ctx, const uint32_t* skl, Cursor& w) {
  Stream& st = ctx->st;
  uint32_t* jv = w.take<uint32_t>(8);
  uint32_t* jr = w.take<uint32_t>(8);
  uint32_t* proj = w.take<uint32_t>(TOM_PROJ_WORDS);
  uint8_t* bytes = w.take<uint8_t>(BSTRIDE);
  copy_h2d(st, jv, skl, 32);
  dev_memset(st, jr, 0, 32);
  launch(st, 1, TomCommitTask{jv, jr, ctx->tg.tab, ctx->tg.tab, proj, ctx->tom, 1});
  launch(st, 1, TraceToE1Task{proj});
  launch_tom_norm(st, proj, nullptr, bytes, 1, 0);
  return bytes;
}
// headers and blocks of rows [b0, b0 + Bc) on the device: device rows through TraceGatherTask; host rows are gathered on
// the host, so that only the header and the block of each row cross PCIe
void trace_gather(zka_ctx* ctx, Cursor& w, const uint8_t* proofs, size_t stride, const uint32_t* len, uint32_t b0, int Bc,
                  uint8_t** hdr, uint8_t** blk, uint8_t** shortrow) {
  Stream& st = ctx->st;
  *hdr = w.take<uint8_t>((size_t)Bc * HEAD_LEN);
  *blk = w.take<uint8_t>((size_t)Bc * TRACE_LEN);
  *shortrow = w.take<uint8_t>(Bc);
  DevBuf& lb = w.next();
  if (is_device_ptr(proofs)) {
    const uint32_t* dl = stage_in(st, lb, len + b0, (size_t)Bc);
    launch(st, Bc, TraceGatherTask{proofs + (size_t)b0 * stride, stride, dl, *hdr, *blk, *shortrow});
    return;
  }
  std::vector<uint32_t> hl((size_t)Bc);
  copy_d2h(st, hl.data(), len + b0, (size_t)Bc * 4);
  sync(st);
  std::vector<uint8_t> h((size_t)Bc * (HEAD_LEN + TRACE_LEN + 1), 0);
  uint8_t *hh = h.data(), *hb = hh + (size_t)Bc * HEAD_LEN, *hs = hb + (size_t)Bc * TRACE_LEN;
  for (int b = 0; b < Bc; b++) {
    const uint8_t* row = proofs + (size_t)(b0 + b) * stride;
    memcpy(hh + (size_t)b * HEAD_LEN, row, std::min<size_t>(HEAD_LEN, stride));
    hs[b] = (hl[b] < (uint32_t)TRACE_LEN || hl[b] > stride) ? 1 : 0;
    if (!hs[b]) memcpy(hb + (size_t)b * TRACE_LEN, row + hl[b] - TRACE_LEN, TRACE_LEN);
  }
  copy_h2d(st, *hdr, h.data(), h.size() - Bc * (size_t)(TRACE_LEN + 1));
  copy_h2d(st, *blk, hb, (size_t)Bc * TRACE_LEN);
  copy_h2d(st, *shortrow, hs, (size_t)Bc);
  sync(st);
}
// the three relations of each staged block: bad[b] (the block does not parse) and rel_ok[3 b + i] on the device
void trace_check(zka_ctx* ctx, const zka_params* P, Cursor& w, int Bc, const uint8_t* y, const uint8_t* msg, const uint8_t* hdr,
                 const uint8_t* blk, const uint8_t* shortrow, uint8_t** bad, uint8_t** rel_ok) {
  Stream& st = ctx->st;
  uint32_t* jv = w.take<uint32_t>((size_t)Bc * 3 * 8);
  uint32_t* jr = w.take<uint32_t>((size_t)Bc * 3 * 8);
  uint32_t* sc = w.take<uint32_t>((size_t)Bc * 4 * 8);
  uint32_t* cproj = w.take<uint32_t>((size_t)Bc * 3 * TOM_PROJ_WORDS);
  *bad = w.take<uint8_t>(Bc);
  *rel_ok = w.take<uint8_t>((size_t)Bc * 3);
  TraceVJobsTask vj{{}, y, msg, hdr, blk, shortrow, jv, jr, sc, *bad};
  memcpy(vj.digest, P->hedge_digest, 32);
  launch(st, Bc, vj);
  launch(st, 3ll * Bc, TomCommitTask{jv, jr, ctx->tg.tab, P->th.tab, cproj, ctx->tom, 1});
  launch(st, 3ll * Bc, TraceVCheckTask{cproj, hdr, blk, y, sc, *rel_ok});
}

// The blocks of rows [b0, b0 + Bc) of a prove call whose untraced pass is complete, appended in the caller's rows
void trace_prove_chunk(zka_ctx* ctx, const zka_params* P, const ProveRows& rows, const uint8_t* y, size_t L, uint32_t b0, int Bc) {
  Stream& st = ctx->st;
  Cursor w(ctx->trace);
  const ProveRows r = rows.at(b0), e = rows.at(b0 + Bc);
  auto stage = [&](auto* p, auto* end) { return stage_in(st, w.next(), p, (size_t)(end - p)); };
  uint8_t* hdr = w.take<uint8_t>((size_t)Bc * HEAD_LEN);
  copy_d2h_2d(st, hdr, HEAD_LEN, r.proofs, rows.proof_stride, HEAD_LEN, Bc);
  const int32_t* d_status = stage(r.status, e.status);
  const uint8_t* d_pk = stage(r.pk, e.pk);
  const uint8_t* d_msg = stage(r.msg_hash, e.msg_hash);
  const uint8_t* d_seeds = stage(r.seeds, e.seeds);
  // tape rows: draw 1 (r) and the four trace draws; a host tape sends only these 160 bytes of each row
  const uint8_t* tape = r.tape;
  size_t ts = rows.tape_stride, r_off = 32, t_off = L;
  DevBuf& tb = w.next();
  if (tape && !is_device_ptr(tape)) {
    uint8_t* d = tb.get<uint8_t>((size_t)Bc * 160);
    copy_d2h_2d(st, d, 160, r.tape + 32, rows.tape_stride, 32, Bc);
    copy_d2h_2d(st, d + 32, 160, r.tape + L, rows.tape_stride, 128, Bc);
    tape = d; ts = 160; r_off = 0; t_off = 32;
  }
  uint32_t* jv = w.take<uint32_t>((size_t)Bc * 5 * 8);
  uint32_t* jr = w.take<uint32_t>((size_t)Bc * 5 * 8);
  uint32_t* sec = w.take<uint32_t>((size_t)Bc * 6 * 8);
  int32_t* tstat = w.take<int32_t>(Bc);
  uint32_t* cproj = w.take<uint32_t>((size_t)Bc * TRACE_PTS * TOM_PROJ_WORDS);
  uint32_t* pproj = w.take<uint32_t>((size_t)Bc * TRACE_PTS * TOM_PROJ_WORDS);
  uint8_t* pbytes = w.take<uint8_t>((size_t)Bc * TRACE_PTS * BSTRIDE);
  uint8_t* blk = w.take<uint8_t>((size_t)Bc * TRACE_LEN);
  launch(st, Bc, TraceJobsTask{d_status, d_pk, tape, ts, r_off, t_off, d_seeds, jv, jr, sec, tstat});
  launch(st, (long long)Bc * TRACE_PTS, TomCommitTask{jv, jr, ctx->tg.tab, P->th.tab, cproj, ctx->tom, 1});
  launch(st, (long long)Bc * TRACE_PTS, TracePointsTask{cproj, sec, y, pproj});
  launch_tom_norm(st, pproj, nullptr, pbytes, (long long)Bc * TRACE_PTS, 0);
  TraceFinishTask fin{{}, y, d_msg, hdr, pbytes, sec, tstat, blk};
  memcpy(fin.digest, P->hedge_digest, 32);
  launch(st, Bc, fin);
  uint8_t* chk = nullptr;
  if (ctx->self_check) {
    uint8_t *bad, *rel;
    trace_check(ctx, P, w, Bc, y, d_msg, hdr, blk, nullptr, &bad, &rel);
    chk = w.take<uint8_t>(Bc);
    launch(st, Bc, TraceSelfCheckTask{bad, rel, tstat, chk});
  }
  // each row's fate is decided on the host: block appended, or the row released like one the prover rejected
  std::vector<int32_t> hts((size_t)Bc), hst((size_t)Bc);
  std::vector<uint32_t> hl((size_t)Bc);
  std::vector<uint8_t> hchk((size_t)Bc, 0);
  copy_d2h(st, hts.data(), tstat, (size_t)Bc * 4);
  copy_d2h(st, hst.data(), r.status, (size_t)Bc * 4);
  copy_d2h(st, hl.data(), r.proof_len, (size_t)Bc * 4);
  if (chk) copy_d2h(st, hchk.data(), chk, (size_t)Bc);
  const bool dev = is_device_ptr(rows.proofs);
  std::vector<uint8_t> hblk(dev ? 0 : (size_t)Bc * TRACE_LEN);
  if (!dev) copy_d2h(st, hblk.data(), blk, hblk.size());
  sync(st);
  std::vector<int64_t> off((size_t)Bc, -1);
  uint64_t failed = 0;
  for (int b = 0; b < Bc; b++) {
    failed += hchk[b] == 2;
    if (hst[b] != ZKA_OK) continue;
    uint8_t* row = r.proofs + (size_t)b * rows.proof_stride;
    if (hts[b] != ZKA_OK) {
      if (dev) dev_memset(st, row, 0, rows.proof_stride); else memset(row, 0, rows.proof_stride);
      hl[b] = 0;
      hst[b] = hts[b];
      continue;
    }
    off[b] = hl[b];
    if (!dev) memcpy(row + hl[b], hblk.data() + (size_t)b * TRACE_LEN, TRACE_LEN);
    hl[b] += TRACE_LEN;
  }
  if (dev) {
    int64_t* d_off = w.take<int64_t>(Bc);
    copy_h2d(st, d_off, off.data(), (size_t)Bc * 8);
    launch(st, Bc, TraceApplyTask{r.proofs, rows.proof_stride, blk, d_off});
  }
  copy_h2d(st, r.proof_len, hl.data(), (size_t)Bc * 4);
  copy_h2d(st, r.status, hst.data(), (size_t)Bc * 4);
  sync(st);
  if (failed) {
    std::lock_guard<std::mutex> g(ctx->stat_mu);
    ctx->self_check_fail += failed;
  }
}

int prove_traced(zka_ctx* ctx, const zka_params* P, uint32_t B, const ProveRows& rows, const uint8_t* ring, uint32_t N,
                 const uint8_t* Y) {
  if (!ctx || !P || !Y || !rows.proofs || !rows.proof_len || !rows.status || !rows.pk || !rows.msg_hash) return ZKA_E_ARG;
  const int S = (int)P->sec_level, n = ceil_log2(N);
  const size_t L = (size_t)32 * prove_draws(S, n, S);
  if (rows.tape && rows.tape_stride < L + 32 * TRACE_DRAWS) return fail(ctx, ZKA_E_ARG, "tape_stride < zka_prove_tape_len + 128");
  if (rows.proof_stride < (size_t)proof_len(S, n, S) + TRACE_LEN)
    return fail(ctx, ZKA_E_ARG, "proof_stride < zka_proof_max_len + zka_trace_len");
  return guarded(ctx, [&] {
    DevBuf ybuf;
    const uint8_t* y = trace_y(ctx, ybuf, Y);
    if (!y) return fail(ctx, ZKA_E_ARG, "Y is not a point of the proof group");
    volatile uint32_t* flags = ctx->progress;
    const uint32_t cap = ctx->progress_cap;
    ctx->progress = nullptr;
    ctx->progress_cap = 0;
    const int rc = prove_batch(ctx, P, B, rows, RingSrc::one(ring, N), 0);
    ctx->progress = flags;
    ctx->progress_cap = cap;
    if (rc || B == 0) return rc;
    // the chunks of the untraced pass (prove_impl's schedule)
    const uint8_t* rnd_in = rows.seeds ? rows.seeds : rows.tape;
    const bool all_dev = is_device_ptr(rows.proofs) && is_device_ptr(rnd_in);
    const std::vector<uint32_t> off =
        chunk_schedule(B, (uint32_t)(all_dev ? ctx->chunk : std::min(ctx->chunk, ctx->host_chunk)), ctx->nlanes, !all_dev);
    for (size_t k = 0; k + 1 < off.size(); k++) {
      for (uint32_t b0 = off[k]; b0 < off[k + 1]; b0 += TRACE_CHUNK)
        trace_prove_chunk(ctx, P, rows, y, L, b0, (int)std::min<uint32_t>(TRACE_CHUNK, off[k + 1] - b0));
      if (flags && k < cap) flags[k] = 1u;
    }
    return 0;
  });
}

int verify_traced(zka_ctx* ctx, const zka_params* P, uint32_t B, const uint8_t* msg_hash, const uint8_t* ring, uint32_t N,
                  const uint8_t* proofs, size_t stride, const uint32_t* proof_len, const uint8_t* tape, size_t tape_stride,
                  const uint8_t* seeds, uint32_t samples, uint8_t* ok, int32_t* status, const uint8_t* Y) {
  if (!ctx || !P || !Y || !msg_hash || !proofs || !proof_len || !ok || !status || (!tape && !seeds)) return ZKA_E_ARG;
  return guarded(ctx, [&] {
    Stream& st = ctx->st;
    DevBuf ybuf, lbuf;
    const uint8_t* y = trace_y(ctx, ybuf, Y);
    if (!y) return fail(ctx, ZKA_E_ARG, "Y is not a point of the proof group");
    if (B == 0) return 0;
    // the untraced verdict of every row's first proof_len - TRACE_LEN bytes
    std::vector<uint32_t> hl(B);
    copy_d2h(st, hl.data(), proof_len, (size_t)B * 4);
    sync(st);
    for (auto& l : hl) l = l >= (uint32_t)TRACE_LEN ? l - TRACE_LEN : 0;
    const uint32_t* base_len = hl.data();
    if (is_device_ptr(proof_len)) {
      uint32_t* d = lbuf.get<uint32_t>(B);
      copy_h2d(st, d, hl.data(), (size_t)B * 4);
      sync(st);
      base_len = d;
    }
    const int rc = seeds ? zka_verify_batch_seeded(ctx, P, B, msg_hash, ring, N, proofs, stride, base_len, seeds, samples, ok, status)
                         : zka_verify_batch_ex(ctx, P, B, msg_hash, ring, N, proofs, stride, base_len, tape, tape_stride, ok, status,
                                               samples);
    if (rc) return rc;
    const Output<uint8_t> oo(ok, 1);
    const Output<int32_t> so(status, 1);
    for (uint32_t b0 = 0; b0 < B; b0 += TRACE_CHUNK) {
      const int Bc = (int)std::min<uint32_t>(TRACE_CHUNK, B - b0);
      Cursor w(ctx->trace);
      uint8_t *hdr, *blk, *sh, *bad, *rel;
      trace_gather(ctx, w, proofs, stride, proof_len, b0, Bc, &hdr, &blk, &sh);
      const uint8_t* d_msg = stage_in(st, w.next(), msg_hash + (size_t)b0 * 32, (size_t)Bc * 32);
      trace_check(ctx, P, w, Bc, y, d_msg, hdr, blk, sh, &bad, &rel);
      uint8_t* d_ok = oo.rows(w.next(), b0, Bc);
      int32_t* d_st = so.rows(w.next(), b0, Bc);
      if (!oo.dev) copy_h2d(st, d_ok, ok + b0, (size_t)Bc);
      if (!so.dev) copy_h2d(st, d_st, status + b0, (size_t)Bc * 4);
      launch(st, Bc, TraceVerdictTask{bad, rel, d_ok, d_st});
      oo.copy_back(st, b0, d_ok, Bc);
      so.copy_back(st, b0, d_st, Bc);
      sync(st);
    }
    return 0;
  });
}
}  // namespace

size_t zka_trace_len(void) { return TRACE_LEN; }

int zka_trace_pubkey(zka_ctx* ctx, const uint8_t sk[32], uint8_t* Y) {
  if (!ctx || !sk || !Y) return ZKA_E_ARG;
  return guarded(ctx, [&] {
    uint32_t skl[8];
    if (!trace_sk(ctx, sk, skl)) return fail(ctx, ZKA_E_ARG, "sk must be in [1, q)");
    Cursor w(ctx->trace);
    const uint8_t* bytes = trace_pubkey_dev(ctx, skl, w);
    copy_d2h(ctx->st, Y, bytes, WP);
    sync(ctx->st);
    return 0;
  });
}

int zka_prove_batch_traced(zka_ctx* ctx, const zka_params* P, uint32_t B, const uint8_t* msg_hash, const uint8_t* sig,
                           const uint8_t* pk, const uint32_t* which, const uint8_t* ring, uint32_t N, const uint8_t* tape,
                           size_t tape_stride, uint8_t* proofs, size_t proof_stride, uint32_t* proof_len_out, int32_t* status,
                           const uint8_t* Y) {
  if (!tape) return ZKA_E_ARG;
  ProveRows r(proofs, proof_stride, proof_len_out, status);
  r.msg_hash = msg_hash; r.sig = sig; r.pk = pk; r.which = which; r.tape = tape; r.tape_stride = tape_stride;
  return prove_traced(ctx, P, B, r, ring, N, Y);
}

int zka_prove_batch_traced_seeded(zka_ctx* ctx, const zka_params* P, uint32_t B, const uint8_t* msg_hash, const uint8_t* sig,
                                  const uint8_t* pk, const uint32_t* which, const uint8_t* ring, uint32_t N, const uint8_t* seeds,
                                  uint8_t* proofs, size_t proof_stride, uint32_t* proof_len_out, int32_t* status, const uint8_t* Y) {
  if (!seeds) return ZKA_E_ARG;
  ProveRows r(proofs, proof_stride, proof_len_out, status);
  r.msg_hash = msg_hash; r.sig = sig; r.pk = pk; r.which = which; r.seeds = seeds;
  return prove_traced(ctx, P, B, r, ring, N, Y);
}

int zka_verify_batch_traced(zka_ctx* ctx, const zka_params* P, uint32_t B, const uint8_t* msg_hash, const uint8_t* ring,
                            uint32_t N, const uint8_t* proofs, size_t proof_stride, const uint32_t* proof_len,
                            const uint8_t* tape, size_t tape_stride, uint8_t* ok, int32_t* status, uint32_t samples,
                            const uint8_t* Y) {
  if (!tape) return ZKA_E_ARG;
  return verify_traced(ctx, P, B, msg_hash, ring, N, proofs, proof_stride, proof_len, tape, tape_stride, nullptr, samples, ok,
                       status, Y);
}

int zka_verify_batch_traced_seeded(zka_ctx* ctx, const zka_params* P, uint32_t B, const uint8_t* msg_hash, const uint8_t* ring,
                                   uint32_t N, const uint8_t* proofs, size_t proof_stride, const uint32_t* proof_len,
                                   const uint8_t* seeds, uint32_t samples, uint8_t* ok, int32_t* status, const uint8_t* Y) {
  if (!seeds) return ZKA_E_ARG;
  return verify_traced(ctx, P, B, msg_hash, ring, N, proofs, proof_stride, proof_len, nullptr, 0, seeds, samples, ok, status, Y);
}

// The opener: the ring's points (ring[j] mod q) g, sorted by a 64-bit key of their encodings (CUB radix sort; std::sort in
// the host simulator), then per row D = C2 - sk C1 and a binary search (TraceFindTask)
int zka_open_batch(zka_ctx* ctx, const zka_params* P, const uint8_t sk[32], uint32_t B, const uint8_t* msg_hash,
                   const uint8_t* ring, uint32_t N, const uint8_t* proofs, size_t proof_stride, const uint32_t* proof_len,
                   uint32_t* index, int32_t* status) {
  if (!ctx || !P || !sk || !msg_hash || !ring || !proofs || !proof_len || !index || !status) return ZKA_E_ARG;
  if (N < 2 || N > (1u << 20)) return fail(ctx, ZKA_E_ARG, "ring size must be in [2, 2^20]");
  return guarded(ctx, [&] {
    uint32_t skl[8];
    if (!trace_sk(ctx, sk, skl)) return fail(ctx, ZKA_E_ARG, "sk must be in [1, q)");
    if (B == 0) return 0;
    Stream& st = ctx->st;
    DevBuf ybuf[4], rin, rjv, rjr, rproj, rbytes, keys, idx, keys2, idx2, tmp;
    Cursor yw(ybuf);
    const uint8_t* y = trace_pubkey_dev(ctx, skl, yw);
    const uint8_t* d_ring = stage_in(st, rin, ring, (size_t)N * 32);
    uint32_t* jv = rjv.get<uint32_t>((size_t)N * 8);
    uint32_t* jr = rjr.get<uint32_t>((size_t)N * 8);
    uint32_t* proj = rproj.get<uint32_t>((size_t)N * TOM_PROJ_WORDS);
    uint8_t* rb = rbytes.get<uint8_t>((size_t)N * BSTRIDE);
    uint64_t* k1 = keys.get<uint64_t>(N);
    uint32_t* i1 = idx.get<uint32_t>(N);
    uint64_t* k2 = keys2.get<uint64_t>(N);
    uint32_t* i2 = idx2.get<uint32_t>(N);
    launch(st, N, TraceRingJobsTask{d_ring, jv, jr});
    launch(st, N, TomCommitTask{jv, jr, ctx->tg.tab, P->th.tab, proj, ctx->tom, 1});
    launch(st, N, TraceToE1Task{proj});
    launch_tom_norm(st, proj, nullptr, rb, (long long)N, 0);
    launch(st, N, TraceKeyTask{rb, k1, i1});
#if defined(ZKA_HOSTSIM)
    {
      std::vector<std::pair<uint64_t, uint32_t>> v(N);
      for (uint32_t j = 0; j < N; j++) v[j] = {k1[j], i1[j]};
      std::sort(v.begin(), v.end());
      for (uint32_t j = 0; j < N; j++) { k2[j] = v[j].first; i2[j] = v[j].second; }
    }
#else
    {
      size_t tb = 0;
      ZK_CUDA_CHECK(cub::DeviceRadixSort::SortPairs(nullptr, tb, k1, k2, i1, i2, (int)N, 0, 64, st.s));
      void* t = tmp.get<uint8_t>(tb);
      ZK_CUDA_CHECK(cub::DeviceRadixSort::SortPairs(t, tb, k1, k2, i1, i2, (int)N, 0, 64, st.s));
    }
#endif
    const Output<uint32_t> io(index, 1);
    const Output<int32_t> so(status, 1);
    for (uint32_t b0 = 0; b0 < B; b0 += TRACE_CHUNK) {
      const int Bc = (int)std::min<uint32_t>(TRACE_CHUNK, B - b0);
      Cursor w(ctx->trace);
      uint8_t *hdr, *blk, *sh, *bad, *rel;
      trace_gather(ctx, w, proofs, proof_stride, proof_len, b0, Bc, &hdr, &blk, &sh);
      const uint8_t* d_msg = stage_in(st, w.next(), msg_hash + (size_t)b0 * 32, (size_t)Bc * 32);
      trace_check(ctx, P, w, Bc, y, d_msg, hdr, blk, sh, &bad, &rel);
      uint32_t* dproj = w.take<uint32_t>((size_t)Bc * TOM_PROJ_WORDS);
      uint8_t* dbytes = w.take<uint8_t>((size_t)Bc * BSTRIDE);
      TraceOpenDTask od{{}, blk, dproj};
      memcpy(od.sk, skl, 32);
      launch(st, Bc, od);
      launch_tom_norm(st, dproj, nullptr, dbytes, Bc, 0);
      uint32_t* d_idx = io.rows(w.next(), b0, Bc);
      int32_t* d_st = so.rows(w.next(), b0, Bc);
      launch(st, Bc, TraceFindTask{bad, rel, dbytes, rb, k2, i2, N, d_idx, d_st});
      io.copy_back(st, b0, d_idx, Bc);
      so.copy_back(st, b0, d_st, Bc);
      sync(st);
    }
    return 0;
  });
}

}  // extern "C"
